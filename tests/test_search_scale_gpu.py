"""Pattern search (K8, csrc/fxg_search.cu) past one work item per warp, past 32 items per query and past 2^21 queries,
against the vectorised reference over the oracle's haystacks (searchscalelib): every hit of Fasta.locate /
locate_approx on a file of 15k items, the first hits of 7,200 slices whose first hit lies at item 31 .. 64, every hit of
Fastq.locate / locate_approx on 11k items and on three truncations of them, and every hit of 2^21 + 1 slices.
searchscalelib states the inputs, test_search_scale_cpu.py that they reach what they aim at.  A failure names the first
differing hit, its work item and where that item sits in the launch, so that the loop that went wrong shows."""
import numpy as np
import pytest

import searchlib as S
import searchscalelib as L
import pyfastx_b200 as pyfastx
from oracle import fxo
from pyfastx_b200 import _cabi

pytestmark = pytest.mark.gpu
PATS = L.patterns()
STRANDS = (("+", 1), ("-", 2), ("both", 3))
BOTH = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS


def check(got, want, label, where, nq):
    """got, want: (query, start, minus[, mismatches]) arrays of a search over nq queries; on a difference, fail with the
    first differing hit of each side described by where(query, start) (a hit a broken kernel left unwritten can hold
    any query)"""
    got = tuple(np.asarray(g, np.int64) for g in got)
    want = tuple(np.asarray(w, np.int64) for w in want)
    n = min(got[0].size, want[0].size)
    diff = np.zeros(n, bool)
    for g, w in zip(got, want):
        diff |= g[:n] != w[:n]
    bad = np.flatnonzero(diff)
    if bad.size == 0 and got[0].size == want[0].size:
        return
    i = int(bad[0]) if bad.size else n

    def show(h):
        if i >= h[0].size:
            return "none (%d hits)" % h[0].size
        q, start = int(h[0][i]), int(h[1][i])
        return "query %d start %d minus %d%s: %s" % (q, start, h[2][i], " mm %d" % h[3][i] if len(h) > 3 else "",
                                                      where(q, start) if 0 <= q < nq and start >= 0 else "not a hit")
    pytest.fail("%s: %d hits, %d expected; first difference at hit %d:\n  got  %s\n  want %s"
                % (label, got[0].size, want[0].size, i, show(got), show(want)))


def fasta_where(item_off, split, nw):
    """a FASTA hit's item it and its place in search_kernel's grid-stride loop: pass it // nw, warp it % nw"""
    def where(q, start):
        it = int(L.hit_items(item_off, split, np.array([q]), np.array([start]))[0])
        return "item %d (item %d of its query; pass it // nw = %d, warp it %% nw = %d, nw = %d)" % (
            it, it - item_off[q], it // nw, it % nw, nw)
    return where


def reads_where(rlen, m):
    """a read hit's item, its tile, and whether the item starts the tile"""
    R = L.reads_items(rlen, m)
    tile_off = np.concatenate([[0], np.cumsum(R["tile"])])

    def where(q, start):
        it = int(L.read_hit_items(R["read_item"], rlen, np.array([q]), np.array([start]))[0])
        t = q // 32
        if it >= tile_off[-1]:
            return "item %d past the last item %d (tile %d)" % (it, tile_off[-1] - 1, t)
        return "item %d of %d in tile %d (items %d .. %d; %s), lanes %d + %d, piece %d" % (
            it, tile_off[-1], t, tile_off[t], tile_off[t + 1] - 1,
            "starts the tile" if it == tile_off[t] else "not the tile's first", R["lane0"][it], R["lanes"][it],
            R["piece"][it])
    return where


def as_tuple(hits, mismatches=False):
    t = (hits["query"], hits["start"], hits["minus"])
    return t + (hits["mismatches"],) if mismatches else t


def located(res):
    return (res[0], res[1], res[2].astype(np.int64)) + tuple(res[3:])


# ---- A: Fasta.locate over 15k items --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fa_a(tmp_path_factory):
    data, kinds, planted, zero_runs = L.fasta_a()
    path = tmp_path_factory.mktemp("a") / "a.fa"
    path.write_bytes(data)
    fa = pyfastx.Fasta(str(path))
    rows = fxo.fasta_scan(data)[0]
    gr = fa._rows
    uni = (gr["pad"][:, 0] & 1) != 0
    assert uni.tolist() == [k["uniform"] for k in kinds] and gr["norm"].tolist() == [k["norm"] for k in kinds]
    assert np.array_equal(gr["slen"], rows["slen"])
    n = len(rows)
    buf, off = L.fasta_haystacks(data, rows, np.arange(n), np.zeros(n, np.int64), rows["slen"])
    rare = L.approx_hits(buf, off, PATS["rare"], 2)
    return dict(data=data, fa=fa, rows=rows, uni=uni, buf=buf, off=off, planted=planted, rare=rare)


def a_where(A, m, eng):
    n = len(A["rows"])
    items, split = L.fasta_items(A["rows"], A["uni"], np.arange(n), np.zeros(n, np.int64), A["rows"]["slen"], m)
    item_off = np.concatenate([[0], np.cumsum(items)])
    return fasta_where(item_off, split, L.fasta_warps(int(item_off[-1]), eng.sm_count))


@pytest.mark.parametrize("name", ["rare", "gaattc", "t", "long"])
def test_fasta_locate(fa_a, name):
    """every occurrence on +, - and both of the rare 16-mer (at piece boundaries, in the last items), of GAATTC, of T
    and of the 1,024-byte pattern in a late item"""
    A = fa_a
    pat = PATS[name]
    both = L.only(A["rare"], 0)[:3] if name == "rare" else L.exact_hits(A["buf"], A["off"], pat)
    where = a_where(A, len(pat), A["fa"]._st.engine)
    for strand, mask in STRANDS:
        check(located(A["fa"].locate(pat, strand)), L.only(both, None, mask), "A %s %s" % (name, strand), where,
              len(A["rows"]))


def test_fasta_locate_approx(fa_a):
    A = fa_a
    where = a_where(A, L.M_RARE, A["fa"]._st.engine)
    for k in (1, 2):
        for strand, mask in STRANDS:
            check(located(A["fa"].locate_approx(PATS["rare"], k, strand)), L.only(A["rare"], k, mask),
                  "A approx k=%d %s" % (k, strand), where, len(A["rows"]))


# ---- B: first hits at item 31 .. 64 ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fa_b(tmp_path_factory):
    data, pat, q, plants = L.first_b()
    path = tmp_path_factory.mktemp("b") / "b.fa"
    path.write_bytes(data)
    fa = pyfastx.Fasta(str(path))
    rows = fxo.fasta_scan(data)[0]
    assert ((fa._rows["pad"][:, 0] & 1) != 0).all()
    buf, off = L.fasta_haystacks(data, rows, np.arange(4), np.zeros(4, np.int64), rows["slen"])
    return dict(data=data, pat=pat, q=q, fa=fa, rows=rows, buf=buf, off=off, whole=L.exact_hits(buf, off, pat))


def test_first_hits_past_32_items(fa_b):
    """Engine.search(first=True) on both strands: 2 * 7,200 (query, strand) warps, so the first-hit loop steps w += nw at
    least twice, and first hits at items 31, 32, 33, 63 and 64 of their query; then every hit of the same slices"""
    B = fa_b
    q, pat, fa = B["q"], B["pat"], B["fa"]
    eng = fa._st.engine
    items, split = L.fasta_items(B["rows"], np.ones(4, bool), q["rid"], q["s"], q["e"], len(pat))
    item_off = np.concatenate([[0], np.cumsum(items)])
    nw = L.fasta_warps(2 * q["rid"].size, eng.sm_count)

    def where(qi, start):
        w = 2 * qi
        rel = start // L.SPIECE
        return ("query %s item %d of %d; first-hit warps w = %d, %d: pass w // nw = %d, nw = %d; b0 block %d"
                % (q["kind"][qi], rel, items[qi], w, w + 1, w // nw, nw, rel // 32))
    every = L.slice_hits(B["whole"], q["rid"], q["s"], q["e"], len(pat))
    got = eng.search(fa._st.dfile, fa._drows, q["rid"], q["s"], q["e"], 0, pat, BOTH, first=True)
    check(as_tuple(got), L.first_hits(every), "B first hits", where, q["rid"].size)
    for strands in (_cabi.SEARCH_PLUS, _cabi.SEARCH_MINUS):
        got = eng.search(fa._st.dfile, fa._drows, q["rid"], q["s"], q["e"], 0, pat, strands, first=True)
        check(as_tuple(got), L.first_hits(L.only(every, None, strands)), "B first hits strands=%d" % strands, where,
              q["rid"].size)
    where_all = fasta_where(item_off, split, L.fasta_warps(int(item_off[-1]), eng.sm_count))
    got = eng.search(fa._st.dfile, fa._drows, q["rid"], q["s"], q["e"], 0, pat, BOTH)
    check(as_tuple(got), every, "B every hit", where_all, q["rid"].size)


def test_sequence_search_past_32_items(fa_b):
    """Sequence.search(p), Sequence.search(p, '-') and `in` on the whole records and on planted slices, against
    str.find on the oracle's haystack"""
    B = fa_b
    q, fa, data, rows = B["q"], B["fa"], B["data"], B["rows"]
    p = B["pat"].decode()
    rng = np.random.default_rng(9)
    pl = np.flatnonzero(q["kind"] == "planted")
    picks = [(r, 0, int(rows["slen"][r])) for r in range(4)]
    picks += [(int(q["rid"][i]), int(q["s"][i]), int(q["e"][i])) for i in rng.choice(pl, 16, replace=False)]
    for r, a, b in picks:
        hay = fxo.subseq(data, rows[r], a, b)
        sub = fa[r] if (a, b) == (0, int(rows["slen"][r])) else fa[r][a:b]
        want = (S.first_position(hay, B["pat"], False), S.first_position(hay, B["pat"], True))
        assert (sub.search(p), sub.search(p, "-")) == want, (r, a, b)
        assert want[0] is not None and (want[0] - 1) // L.SPIECE >= 31
        rc = S.revcomp(B["pat"])
        assert (p in sub) is True and (rc.decode() in sub) == (rc in hay)


# ---- C: Fastq.locate over 11k items ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fq_c(tmp_path_factory):
    data, tiles, planted = L.fastq_c()
    d = tmp_path_factory.mktemp("c")
    path = d / "c.fq"
    path.write_bytes(data)
    fq = pyfastx.Fastq(str(path))
    rows = fxo.fastq_scan(data)[0]
    assert len(fq) == len(rows) and np.array_equal(fq._rows["rlen"], rows["rlen"])
    buf, off = L.read_haystacks(data, rows)
    rare = L.approx_hits(buf, off, PATS["rare"], 2)
    exact = {name: (L.only(rare, 0)[:3] if name == "rare" else L.exact_hits(buf, off, pat)) for name, pat in PATS.items()}
    return dict(data=data, dir=d, fq=fq, rows=rows, rare=rare, exact=exact)


@pytest.mark.parametrize("name", ["rare", "gaattc", "t", "long"])
def test_fastq_locate(fq_c, name):
    C = fq_c
    pat = PATS[name]
    where = reads_where(C["rows"]["rlen"], len(pat))
    for strand, mask in STRANDS:
        check(located(C["fq"].locate(pat, strand)), L.only(C["exact"][name], None, mask), "C %s %s" % (name, strand),
              where, len(C["rows"]))


def test_fastq_locate_approx(fq_c):
    C = fq_c
    where = reads_where(C["rows"]["rlen"], L.M_RARE)
    for k in (1, 2):
        for strand, mask in STRANDS:
            check(located(C["fq"].locate_approx(PATS["rare"], k, strand)), L.only(C["rare"], k, mask),
                  "C approx k=%d %s" % (k, strand), where, len(C["rows"]))


@pytest.mark.parametrize("drop", [1, 37, 301])
def test_fastq_truncated(fq_c, drop):
    """C without its last `drop` reads: another item total, so every warp's range and the last one's length move.
    The reads kept are the same reads (checked against the oracle's scan), so their hits are the full file's."""
    C = fq_c
    rows = C["rows"]
    n = len(rows) - drop
    cut = int(rows["qoff"][n - 1] + rows["rlen"][n - 1]) + 1
    data = C["data"][:cut]
    assert data.endswith(b"\n") and np.array_equal(fxo.fastq_scan(data)[0], rows[:n])
    path = C["dir"] / ("c%d.fq" % drop)
    path.write_bytes(data)
    fq = pyfastx.Fastq(str(path))
    assert len(fq) == n

    def keep(h):
        k = h[0] < n
        return tuple(x[k] for x in h)
    for name, pat in PATS.items():
        check(located(fq.locate(pat, "both")), keep(C["exact"][name]), "C[:-%d] %s" % (drop, name),
              reads_where(rows["rlen"][:n], len(pat)), n)
    check(located(fq.locate_approx(PATS["rare"], 1, "both")), keep(L.only(C["rare"], 1)), "C[:-%d] approx" % drop,
          reads_where(rows["rlen"][:n], L.M_RARE), n)


# ---- D: 2^21 + 1 one-item slices -------------------------------------------------------------------------------------
def test_slices_past_2_21(fa_a):
    """Engine.search (every hit, both strands) and Engine.search_approx (k = 1) on 2^21 + 1 slices of one item each:
    the item prefix and the hit prefix take a second chunk of ps_scan_sums"""
    A = fa_a
    fa = A["fa"]
    eng = fa._st.engine
    rid, s, e = L.slices_d(A["rows"], A["uni"], A["planted"])
    nw = L.fasta_warps(rid.size, eng.sm_count)

    def where(q, start):
        return "item %d (pass it // nw = %d, warp it %% nw = %d, nw = %d)" % (q, q // nw, q % nw, nw)
    got = eng.search(fa._st.dfile, fa._drows, rid, s, e, 0, PATS["rare"], BOTH)
    check(as_tuple(got), L.slice_hits(L.only(A["rare"], 0)[:3], rid, s, e, L.M_RARE), "D exact", where, rid.size)
    got = eng.search_approx(fa._st.dfile, fa._drows, rid, s, e, 0, PATS["rare"], 1, BOTH)
    check(as_tuple(got, True), L.slice_hits(L.only(A["rare"], 1), rid, s, e, L.M_RARE), "D approx k=1", where, rid.size)
