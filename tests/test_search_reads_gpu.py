"""Pattern search in FASTQ reads on the GPU against the oracle-read expectation: full hit lists of Fastq.locate on every
strand setting, on the layouts that decide which bytes a read's haystack is and how reads become work items."""
import ctypes as C
import gzip

import numpy as np
import pytest

import readsearchlib as R
import searchlib as S
import pyfastx_b200 as pyfastx
from pyfastx_b200 import _cabi, synth

pytestmark = pytest.mark.gpu
PIECE, CAP = _cabi.SEARCH_PIECE, _cabi.SEARCH_MAX_PATTERN
STRANDS = (("+", 1), ("-", 2), ("both", 3))


def write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def rand_seq(n, seed, alphabet=b"ACGT"):
    rng = np.random.default_rng(seed)
    return bytes(np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), n)])


def record(name, seq, qual=None, eol=b"\n"):
    return b"@" + name + eol + seq + eol + b"+" + eol + (b"I" * len(seq) if qual is None else qual) + eol


def locate_list(fq, pat, strand):
    rid, start, minus = fq.locate(pat, strand)
    assert rid.dtype == np.int64 and start.dtype == np.int64 and minus.dtype == bool
    key = rid * (1 << 40) + start * 2 + minus
    assert np.all(np.diff(key) > 0)                                            # strictly (read, start, minus) ordered
    return list(zip(rid.tolist(), start.tolist(), minus.astype(int).tolist()))


def check(fq, hays, pats, strands=STRANDS):
    for pat in pats:
        pb = pat.encode("latin-1") if isinstance(pat, str) else pat
        for strand, mask in strands:
            assert locate_list(fq, pat, strand) == S.expected_hits(hays, pb, mask), (pat[:40], strand)


def open_checked(tmp_path, name, data):
    fq = pyfastx.Fastq(write(tmp_path, name, data))
    rows, hays = R.read_haystacks(data)
    assert len(fq) == len(rows)
    return fq, hays


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"])
def test_read_lengths_lf_and_crlf(tmp_path, eol):
    lengths = [0, 1, 4, 5, 16, 17, 150, 151, PIECE - 1, PIECE, PIECE + 1, 2 * PIECE + 3, 0, 150, 1]
    seqs = [rand_seq(n, 50 + i) for i, n in enumerate(lengths)]
    data = b"".join(record(b"r%d" % i, s, rand_seq(len(s), 900 + i), eol) for i, s in enumerate(seqs))
    fq, hays = open_checked(tmp_path, "len%d.fq" % len(eol), data)
    assert hays == seqs
    pats = ["T", "AC", "GATC"]
    for m in (1, 4, 5, 17, 150):
        for s in seqs:
            if len(s) >= m:
                pats += [s[:m], s[-m:], s[len(s) // 2 - m // 2:][:m]]              # read start, read end, middle
    pats.append(seqs[11][PIECE - 600:PIECE + 424])                              # CAP bytes across a piece boundary
    check(fq, hays, pats)


@pytest.mark.parametrize("m", [1, 2, 17, CAP])
def test_long_read_piece_boundaries(tmp_path, m):
    """a match starting at every offset in [k * PIECE - m + 1, k * PIECE] of a long read, k = 1, 2, 3"""
    n = 3 * PIECE + CAP + 777
    long_a, long_b = rand_seq(n, 300 + m), rand_seq(n - 5, 400 + m)
    short = [rand_seq(150, 500 + i) for i in range(5)]
    data = (record(b"s0", short[0]) + record(b"la", long_a) + record(b"s1", short[1]) + record(b"s2", short[2]) +
            record(b"lb", long_b) + record(b"s3", short[3]))
    fq, hays = open_checked(tmp_path, "long%d.fq" % m, data)
    for k in (1, 2, 3):
        for o in range(k * PIECE - m + 1, k * PIECE + 1):
            pat = long_a[o:o + m]
            hits = locate_list(fq, pat, "both")
            assert hits == S.expected_hits(hays, pat, 3), (k, o)
            assert (1, o, 0) in hits
    for o in (PIECE - m + 1, 2 * PIECE, n - m):
        check(fq, hays, [long_a[o:o + m], long_b[o - 5:o - 5 + m]], STRANDS[:2])


def test_boundaries_never_match(tmp_path):
    """names, sequences and qualities of A/C/G/T letters; patterns that occur only across a sequence line's end, a
    quality line's end into the next name, or across two reads' sequences"""
    for eol in (b"\n", b"\r\n"):
        n = 40
        names = [rand_seq(10, 10 + i) for i in range(n)]
        seqs = [rand_seq(20 + (i % 7) * 31, 100 + i) for i in range(n)]
        quals = [rand_seq(len(s), 200 + i) for i, s in enumerate(seqs)]
        data = b"".join(record(nm, s, q, eol) for nm, s, q in zip(names, seqs, quals))
        fq, hays = open_checked(tmp_path, "b%d.fq" % len(eol), data)
        pats = []
        for i in range(n - 1):
            pats += [seqs[i][-3:] + eol, seqs[i][-3:] + eol + b"+", seqs[i][-4:] + eol + b"+" + eol + quals[i][:4],
                     quals[i][-4:] + eol + b"@" + names[i + 1][:5], seqs[i][-8:] + seqs[i + 1][:8],
                     seqs[i][-1:] + seqs[i + 1][:14], seqs[i][-3:] + b"\r"]
        for pat in pats:
            pat = bytes(pat)
            assert S.expected_hits(hays, pat, 3) == [], pat
            for strand, _ in STRANDS:
                assert locate_list(fq, pat, strand) == [], (pat, strand)
        # the same reads do match inside themselves
        check(fq, hays, [seqs[3][-8:], seqs[4][:8], seqs[7][5:19]])


def test_tiles_rounds_and_order(tmp_path):
    """reads around every multiple of the tile size (32), a long read in the middle of a tile, two long reads next to
    each other, and tiles whose reads need several staging rounds"""
    rng = np.random.default_rng(7)
    lens = [int(x) for x in rng.integers(100, 300, 200)]
    lens[40] = 3 * PIECE + 11                                                   # middle of the second tile
    lens[70] = lens[71] = 2 * PIECE + 1                                         # next to each other
    lens[128:160] = [PIECE] * 32                                                # one read per staging round
    lens[160:192] = [int(x) for x in rng.integers(600, 1200, 32)]
    seqs = [rand_seq(n, 1000 + i) for i, n in enumerate(lens)]
    body = [record(b"q%d" % i, s) for i, s in enumerate(seqs)]
    pats = ["GAATTC", "ACGT", "TTT", "G", seqs[40][PIECE - 3:PIECE + 9].decode(), seqs[71][:30].decode(),
            seqs[150][-20:].decode(), seqs[31][-12:].decode(), seqs[32][:12].decode()]
    for count in (1, 31, 32, 33, 63, 64, 65, 96, 200):
        data = b"".join(body[:count])
        fq, hays = open_checked(tmp_path, "t%d.fq" % count, data)
        check(fq, hays, pats if count == 200 else pats[:4] + pats[7:])


def test_raw_semantics(tmp_path):
    lower = rand_seq(700, 3, b"acgtnACGTN")
    iupac = rand_seq(500, 4, b"ACGTRYKMBVDHNUacgtrykmbvdhnu")
    high = bytes(rand_seq(300, 5, b"ACGT\x80\xe9\xff"))
    seqs = [b"TTAC GTAA", b"AC\tGTAC GT", lower, iupac, high, b"TTGAATTCAAGAATTCGGATCC" * 20, b"A" * 5000,
            b"AAAACAAAA" * 10, b"A" * CAP, b"A" * (CAP - 1)]
    data = b"".join(record(b"x%d" % i, s) for i, s in enumerate(seqs))
    fq, hays = open_checked(tmp_path, "raw.fq", data)
    assert hays == seqs
    assert locate_list(fq, "AC GT", "+") == [(0, 2, 0), (1, 5, 0)]               # a space is part of a read
    assert locate_list(fq, b"AC\tGT", "+") == [(1, 0, 0)]
    assert locate_list(fq, "ACGT", "both") == S.expected_hits(hays, b"ACGT", 3)
    check(fq, hays, ["AC GT", "C\tG", "acgt", "ACGT", "gaattc", "GAATTC", "GGATCC", "RYKM", "n", "N", lower[100:130],
                     iupac[200:210], high[10:25], b"\xe9", b"\x80\xff", "AAAA", "A" * CAP, "A", "TTTT"])
    rid, start, minus = fq.locate("AAAA", "both")
    assert int(((rid == 6) & ~minus).sum()) == 5000 - 3 and int(((rid == 6) & minus).sum()) == 0
    rid, _, _ = fq.locate("A" * CAP, "+")
    assert rid.tolist().count(6) == 5000 - CAP + 1 and rid.tolist().count(8) == 1 and 9 not in rid.tolist()


def test_every_way_of_opening_gives_the_same_hits(tmp_path):
    data = synth.synth_fastq(500, seed=31, read_len=151)
    pats = ["GAATTC", "ACGTAC", "T", data[1000:1012].decode()]
    L = _cabi.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.c_void_p(), C.c_int64(0)
    _cabi.check(L.fxg_bgzf_compress_host(a.ctypes.data, a.size, 6, C.byref(out), C.byref(n)))
    comp = C.string_at(out.value, n.value)
    L.fxg_free_host(out)
    assert gzip.decompress(comp) == data
    _, hays = R.read_haystacks(data)
    plain = pyfastx.Fastq(write(tmp_path, "p.fq", data))
    again = pyfastx.Fastq(str(tmp_path / "p.fq"))                              # loads the .fxi written by the first open
    gz = pyfastx.Fastq(write(tmp_path, "p.fq.gz", comp))
    assert again._n_lines is None and gz.is_gzip and gz._st.bgzf_members > 1
    for pat in pats:
        exp = S.expected_hits(hays, pat.encode(), 3)
        assert locate_list(plain, pat, "both") == exp
        assert locate_list(again, pat, "both") == exp
        assert locate_list(gz, pat, "both") == exp
    # a trailing partial record is not a read: not searched
    part = data + b"@tail\nGAATTCGAATTC\n+\n"
    fq, hays2 = open_checked(tmp_path, "part.fq", part)
    assert len(fq) == 500 and hays2 == hays
    check(fq, hays2, ["GAATTCGAATTC", "GAATTC"])
    # no complete read at all
    fq = pyfastx.Fastq(write(tmp_path, "none.fq", b"@only\nACGTACGT\n+\n"))
    assert len(fq) == 0
    rid, start, minus = fq.locate("ACGT", "both")
    assert rid.size == start.size == minus.size == 0
    assert rid.dtype == np.int64 and start.dtype == np.int64 and minus.dtype == bool


def test_arguments(tmp_path):
    data = b"".join(record(b"a%d" % i, rand_seq(90, 60 + i)) for i in range(50))
    fq, hays = open_checked(tmp_path, "args.fq", data)
    for strand, _ in STRANDS:
        assert locate_list(fq, "GATC", strand) == locate_list(fq, b"GATC", strand)
        assert locate_list(fq, "GATC", strand) == locate_list(fq, bytearray(b"GATC"), strand)
    for bad in ("", b"", "A" * (CAP + 1)):
        with pytest.raises(ValueError):
            fq.locate(bad)
    for bad in ("x", "+-", None):
        with pytest.raises(ValueError):
            fq.locate("ACGT", strand=bad)
    rid, start, minus = fq.locate("ACG", "both")
    for k in range(rid.size):
        seq = fq[int(rid[k])].seq
        want = "ACG" if not minus[k] else "CGT"
        assert seq[int(start[k]):int(start[k]) + 3] == want


def test_random_patterns(tmp_path):
    data = synth.synth_fastq(3000, seed=20240602)
    fq, hays = open_checked(tmp_path, "rand.fq", data)
    eng = fq._st.engine
    rng = np.random.default_rng(99)
    for t in range(300):
        kind = t % 3
        if kind < 2:
            h = hays[int(rng.integers(0, len(hays)))]
            a = int(rng.integers(0, len(h)))
            pat = h[a:a + int(rng.integers(1, 41))]
            if kind == 1:
                pat = S.revcomp(pat)
        else:
            pat = rand_seq(int(rng.integers(14, 30)), 5000 + t)
        mask = (1, 2, 3)[(t // 3) % 3]
        got = eng.search_reads(fq._st.dfile, fq._drows, pat, mask)
        assert list(zip(got["query"].tolist(), got["start"].tolist(), got["minus"].tolist())) == \
            S.expected_hits(hays, pat, mask), (t, pat)
