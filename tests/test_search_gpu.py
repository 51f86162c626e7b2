"""Pattern search (K8) on the GPU against the oracle-haystack expectation: full hit lists of Fasta.locate and of
Engine.search on slices, Sequence.search and `in`, on the layouts that decide which bytes a query's haystack is."""
import ctypes as C
import gzip
import os

import numpy as np
import pytest

import goldenlib as G
import searchlib as S
import pyfastx_b200 as pyfastx
from pyfastx_b200 import _cabi, synth
from oracle import fxo

pytestmark = pytest.mark.gpu
PIECE, CAP = _cabi.SEARCH_PIECE, _cabi.SEARCH_MAX_PATTERN
BOTH = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def rand_seq(n, seed, alphabet=b"ACGT"):
    rng = np.random.default_rng(seed)
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def wrap(seq, width, eol=b"\n"):
    return b"".join(seq[i:i + width] + eol for i in range(0, len(seq), width))


def hit_list(hits):
    return list(zip(hits["query"].tolist(), hits["start"].tolist(), hits["minus"].tolist()))


def locate_list(fa, pat, strand):
    rid, start, minus = fa.locate(pat, strand)
    assert rid.dtype == np.int64 and start.dtype == np.int64 and minus.dtype == bool
    return list(zip(rid.tolist(), start.tolist(), minus.astype(int).tolist()))


def check_file(tmp_path, data, patterns, uppercase=False, name="x.fa"):
    """locate on both strands, Sequence.search on both strands and `in` for every record, against the oracle"""
    fa = pyfastx.Fasta(write(tmp_path, name, data), uppercase=uppercase)
    _, hays = S.whole_records(data, upper=uppercase)
    for pat in patterns:
        pb = pat.encode("latin-1")
        for strand, mask in (("+", 1), ("-", 2), ("both", 3)):
            assert locate_list(fa, pat, strand) == S.expected_hits(hays, pb, mask), (pat, strand)
        for i, h in enumerate(hays):
            sq = fa[i]
            assert sq.search(pat) == S.first_position(h, pb, False), (pat, i)
            assert sq.search(pat, "-") == S.first_position(h, pb, True), (pat, i)
            assert (pat in sq) == (pb in h)
    return fa, hays


def test_matches_across_lf_and_crlf_breaks(tmp_path):
    seqs = [rand_seq(n, 10 + n) for n in (1000, 333, 12345)]
    for eol in (b"\n", b"\r\n"):
        data = b"".join(b">r%d\n".replace(b"\n", eol) % i + wrap(s, 60, eol) for i, s in enumerate(seqs))
        # patterns cut across line ends (60 bases per line) and inside lines
        pats = [seqs[0][55:70].decode(), seqs[2][119:121].decode(), seqs[2][5999:6030].decode(), seqs[1][-7:].decode(),
                "ACG", "T"]
        check_file(tmp_path, data, pats, name="crlf.fa" if len(eol) == 2 else "lf.fa")


@pytest.mark.parametrize("m", [1, 2, 17, CAP])
def test_piece_boundaries_and_slice_ends(tmp_path, m):
    """a match starting at every offset in [PIECE - m + 1, PIECE] of the first piece; a match that straddles a slice's
    end does not count"""
    seq = rand_seq(3 * PIECE + 777, 99 + m)
    data = b">a\n" + wrap(seq, 70) + b">b\n" + wrap(seq[:500], 70)
    fa = pyfastx.Fasta(write(tmp_path, "p.fa", data))
    rows, _, _ = fxo.fasta_scan(data)
    eng, slen = fa._st.engine, len(seq)
    ref = S.haystacks(data, rows, [0], [0], [slen])[0]
    assert ref == seq
    for o in range(PIECE - m + 1, PIECE + 1):
        pat = seq[o:o + m]
        qs = [(0, 0, slen), (0, 0, o + m - 1), (0, 0, o + m), (0, o, slen), (0, 1, o + m), (0, o + 1, slen), (1, 0, 500)]
        rid, s, e = (np.array(x, dtype=np.int64) for x in zip(*qs))
        hays = [seq[a:b] if r == 0 else seq[:500] for r, a, b in qs]
        got = eng.search(fa._st.dfile, fa._drows, rid, s, e, 0, pat, BOTH)
        exp = S.expected_hits(hays, pat, 3)
        assert hit_list(got) == exp, o
        assert (0, o, 0) in exp and (1, o, 0) not in exp and (2, o, 0) in exp   # query 1 ends one byte inside the match
        # the first hit of each (query, strand), both strands in one call: merged in (start, minus) order per query
        first = eng.search(fa._st.dfile, fa._drows, rid, s, e, 0, pat, BOTH, first=True)
        assert hit_list(first) == S.first_hits(exp), o
    # the slices of the first query set, through the oracle's own extraction
    hs = S.haystacks(data, rows, [0, 0, 0], [0, 1, PIECE], [PIECE + 5, slen, slen])
    assert hs == [seq[:PIECE + 5], seq[1:], seq[PIECE:]]


def test_irregular_records(tmp_path):
    long_line = rand_seq(2 * PIECE + 300, 5)
    odd = rand_seq(900, 6)
    recs = [
        b">blank\n" + wrap(odd[:300], 60) + b"\n" + wrap(odd[300:], 60),            # blank line: norm = 0
        b">odd\n" + odd[:100] + b"\n" + odd[100:130] + b"\n" + wrap(odd[130:], 100),  # odd line lengths
        b">oneline\n" + long_line + b"\n",                                         # a line longer than a piece
        b">wide\n" + wrap(long_line, PIECE + 33),                                  # uniform lines longer than a piece
        b">short\nACG\n",                                                          # shorter than most patterns
        b">empty\n",
        b">tail\n" + wrap(odd, 61)[:-1],                                           # no trailing newline
    ]
    data = b"".join(recs)
    pats = [odd[290:320].decode(), odd[95:140].decode(), long_line[PIECE - 10:PIECE + 10].decode(),
            long_line[PIECE + 20:PIECE + 60].decode(), "ACG", "ACGT", "G", odd[-5:].decode()]
    check_file(tmp_path, data, pats)


@pytest.mark.parametrize("m", [1, 17, CAP])
def test_long_irregular_records_stream_window_by_window(tmp_path, m):
    """records that are not cut into pieces and are longer than 3 windows: a norm = 0 record (a blank line in the middle)
    and a norm = 1 record whose one odd line is not the last (slices there take the slice formula, whole records the
    strip).  Matches around every window boundary k * PIECE of the haystack, whole records and slices with s > 0."""
    n = 3 * PIECE + CAP + 777
    a, b = rand_seq(n, 300 + m), rand_seq(6045 + 60 * 122, 400 + m)
    data = (b">blank\n" + wrap(a[:6000], 60) + b"\n" + wrap(a[6000:], 60) +
            b">odd1\n" + wrap(b[:6000], 60) + b[6000:6045] + b"\n" + wrap(b[6045:], 60))
    fa = pyfastx.Fasta(write(tmp_path, "w.fa", data))
    rows, _, _ = fxo.fasta_scan(data)
    assert rows["norm"].tolist() == [0, 1] and (fa._rows["pad"][:, 0] & 1).tolist() == [0, 0]
    slen = rows["slen"].tolist()
    assert min(slen) >= 3 * PIECE + CAP
    eng = fa._st.engine
    for r in (0, 1):
        hay = S.haystacks(data, rows, [r], [0], [slen[r]])[0]
        for k in (1, 2, 3):
            for o in sorted({k * PIECE - m + 1, k * PIECE - m // 2, k * PIECE - 1, k * PIECE}):
                pat = hay[o:o + m]
                L = slen[r]
                qs = [(r, 0, L), (r, 1, L), (r, 333, L - 5), (r, PIECE + 7, L), (r, 0, o + m - 1), (r, 0, o + m),
                      (1 - r, 0, slen[1 - r])]
                rid, s, e = (np.array(x, dtype=np.int64) for x in zip(*qs))
                hays = S.haystacks(data, rows, rid, s, e)
                exp = S.expected_hits(hays, pat, 3)
                assert (0, o, 0) in exp
                got = eng.search(fa._st.dfile, fa._drows, rid, s, e, 0, pat, BOTH)
                assert hit_list(got) == exp, (r, k, o)
                first = eng.search(fa._st.dfile, fa._drows, rid, s, e, 0, pat, BOTH, first=True)
                assert hit_list(first) == S.first_hits(exp), (r, k, o)
                for (_, qa, qb), h in zip(qs[1:4], hays[1:4]):
                    sub = fa[r][qa:qb]
                    ps = pat.decode()
                    assert (sub.search(ps), sub.search(ps, "-")) == (S.first_position(h, pat, False),
                                                                     S.first_position(h, pat, True)), (r, k, o, qa)
        pat = hay[PIECE - 3:PIECE - 3 + m]
        assert locate_list(fa, pat.decode(), "both") == S.expected_hits(S.whole_records(data)[1], pat, 3)


def test_case_iupac_and_palindromes(tmp_path):
    lower = rand_seq(5000, 7, b"acgtnACGTN")
    iupac = rand_seq(3000, 8, b"ACGTRYKMBVDHNUacgtrykmbvdhnu")
    data = b">low\n" + wrap(lower, 80) + b">iupac\n" + wrap(iupac, 50) + b">pal\n" + wrap(b"TTGAATTCAAGAATTCGGATCC" * 40, 33)
    pats = ["GAATTC", "gaattc", "ACGT", "acgt", lower[1000:1012].decode(), iupac[700:709].decode(), "RYKM", "ggatcc",
            "GGATCC", "N", "n"]
    for up in (False, True):
        check_file(tmp_path, data, pats, uppercase=up, name="case%d.fa" % up)


def test_overlapping_runs_and_one_letter(tmp_path):
    runs = b"A" * 5000 + b"C" * 7 + b"A" * 9000 + b"GT" * 3000
    data = b">runs\n" + wrap(runs, 80) + b">mix\n" + wrap(rand_seq(20000, 11), 80)
    fa, hays = check_file(tmp_path, data, ["AAAA", "A", "T", "AC", "GTGTG", "A" * CAP])
    rid, start, minus = fa.locate("A", "both")
    assert rid.size == sum(h.count(b"A") + h.count(b"T") for h in hays)
    assert np.all(np.diff(rid * (1 << 40) + start * 2 + minus) > 0)             # strictly (row, start, minus) ordered


def test_pattern_edge_cases(tmp_path):
    data = b">a\nACGTACGT\nACGT\n>b\nGGCC\n>c\n" + wrap(rand_seq(3000, 12), 60)
    fa = pyfastx.Fasta(write(tmp_path, "e.fa", data))
    s = fa["a"]
    assert fa.locate("T\nA")[0].size == 0 and s.search("T\nA") is None and "T\nA" not in s
    assert s.search("") == 1 and s.search("", "-") == 1 and "" in s
    assert fa["b"][2:2].search("") == 1 and fa["b"][2:2].search("G") is None
    assert s.search("AC€GT") is None and "€" not in s
    with pytest.raises(UnicodeEncodeError):                                    # as the host path raises today
        s.search("€", "-")
    for bad in ("", "A" * (CAP + 1)):
        with pytest.raises(ValueError):
            fa.locate(bad)
    with pytest.raises(ValueError):
        fa.locate("ACGT", strand="x")
    c = fa["c"]
    over = c.seq[100:100 + CAP + 1]                                            # over the cap: the host scan
    k = c.seq.find(pyfastx.reverse_complement(over))
    assert c.search(over) == 101 and c.search(over, "-") == (k + 1 if k >= 0 else None)
    assert over in c
    assert fa.locate(b"ACGT")[0].tolist() == fa.locate("ACGT")[0].tolist()
    assert s.search("GTAC") == 3 and s.search("GTAC", "-") == 3


def test_bgzf_copy_gives_identical_hits(tmp_path):
    data = synth.synth_fasta(60, seed=31, min_len=3000, max_len=9000, width=70)
    L = _cabi.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.c_void_p(), C.c_int64(0)
    _cabi.check(L.fxg_bgzf_compress_host(a.ctypes.data, a.size, 6, C.byref(out), C.byref(n)))
    comp = C.string_at(out.value, n.value)
    L.fxg_free_host(out)
    plain = pyfastx.Fasta(write(tmp_path, "p.fa", data))
    gz = pyfastx.Fasta(write(tmp_path, "p.fa.gz", comp))
    assert gz.is_gzip and gz._st.bgzf_members > 1 and gzip.decompress(comp) == data
    _, hays = S.whole_records(data)
    for pat in ("GAATTC", "ACGTAC", data[5000:5020].decode(), "T"):
        exp = S.expected_hits(hays, pat.encode(), 3)
        assert locate_list(plain, pat, "both") == exp and locate_list(gz, pat, "both") == exp


def test_random_slices_match_str_find(tmp_path):
    data = synth.synth_fasta(200, seed=77, min_len=2000, max_len=12000, width=75)
    fa = pyfastx.Fasta(write(tmp_path, "r.fa", data))
    slen = fa._rows["slen"]
    rng = np.random.default_rng(4242)
    for strand in ("+", "-"):
        for _ in range(1000):
            i = int(rng.integers(0, len(slen)))
            a = int(rng.integers(0, slen[i]))
            b = int(rng.integers(a, slen[i] + 1))
            sub = fa[i][a:b]
            seq = sub.seq
            if rng.random() < 0.7 and b > a:                                   # mostly patterns that occur
                k = int(rng.integers(a, b)) - a
                q = seq[k:k + int(rng.integers(1, 40))]
                if strand == "-":
                    q = pyfastx.reverse_complement(q)
            else:
                q = "".join(rng.choice(list("ACGT"), int(rng.integers(1, 12))))
            target = q if strand == "+" else pyfastx.reverse_complement(q)
            k = seq.find(target)
            assert sub.search(q, strand) == (k + 1 if k >= 0 else None), (i, a, b, q, strand)
