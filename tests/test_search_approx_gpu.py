"""Search with mismatches on the GPU against the numpy expectation over the oracle's haystacks: full hit lists, mismatch
counts included, of Fasta.locate_approx, Fastq.locate_approx and Engine.search_approx on slices, for k in {0, 1, 2, 3,
m - 1} on every strand setting, on the layouts that decide which bytes a haystack is and how it becomes work items."""
import ctypes as C
import gzip

import numpy as np
import pytest

import approxlib as A
import readsearchlib as R
import searchlib as S
import pyfastx_b200 as pyfastx
from pyfastx_b200 import _cabi, synth
from oracle import fxo

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


def wrap(seq, width, eol=b"\n"):
    return b"".join(seq[i:i + width] + eol for i in range(0, len(seq), width))


def fq_record(name, seq, qual=None, eol=b"\n"):
    return b"@" + name + eol + seq + eol + b"+" + eol + (b"I" * len(seq) if qual is None else qual) + eol


def ks(m):
    return sorted({k for k in (0, 1, 2, 3, m - 1) if 0 <= k < m})


def hit_list(hits):
    return list(zip(hits["query"].tolist(), hits["start"].tolist(), hits["minus"].tolist(), hits["mismatches"].tolist()))


def approx_list(obj, pat, k, strand):
    rid, start, minus, mm = obj.locate_approx(pat, k, strand)
    assert rid.dtype == np.int64 and start.dtype == np.int64 and minus.dtype == bool and mm.dtype == np.int32
    key = rid * (1 << 40) + start * 2 + minus
    assert np.all(np.diff(key) > 0)                                            # strictly (id, start, minus) ordered
    assert np.all((mm >= 0) & (mm <= k))
    return list(zip(rid.tolist(), start.tolist(), minus.astype(int).tolist(), mm.tolist()))


def check(obj, hays, pats, kset=None, strands=STRANDS):
    """every k of kset (default ks(m)) on every strand setting against approxlib"""
    for pat in pats:
        pb = pat.encode("latin-1") if isinstance(pat, str) else bytes(pat)
        counts = A.strand_counts(hays, pb)
        for k in (kset if kset is not None else ks(len(pb))):
            if k >= len(pb):
                continue
            for strand, mask in strands:
                assert approx_list(obj, pat, k, strand) == A.expected_from_counts(counts, k, mask), (pb[:40], k, strand)


def variant(pat, d, seed):
    """pat with exactly d substituted bytes (A/C/G/T for A/C/G/T), its first and last byte among them when d allows"""
    rng = np.random.default_rng(seed)
    m = len(pat)
    pos = [0, m - 1][:d] + [int(x) for x in rng.permutation(np.arange(1, m - 1))[:max(d - 2, 0)]]
    v = bytearray(pat)
    for j in pos:
        v[j] = b"ACGT"[(b"ACGT".index(v[j]) + 1 + int(rng.integers(0, 3))) % 4]
    assert sum(a != b for a, b in zip(v, pat)) == d
    return bytes(v)


def planted(n, pat, offsets, seed):
    """one record per offset: random bases with a variant of pat (plus strand on even records, its reverse complement on
    odd ones) of 0 .. 4 substitutions at that offset"""
    rc = S.revcomp(pat)
    out = []
    for i, o in enumerate(offsets):
        s = bytearray(rand_seq(n, seed + i))
        p = rc if i & 1 else pat
        s[o:o + len(p)] = variant(p, i % 5 if i % 5 < len(p) else 0, seed + 7 * i)
        out.append(bytes(s))
    return out


def around_pieces(m, n):
    """start offsets around the piece (and streamed-window) boundaries k * PIECE that fit a record of n bases"""
    offs = set()
    for k in (1, 2):
        b = k * PIECE
        offs |= {b - m - 1, b - m, b - m + 1, b - m + 2, b - m // 2, b - 2, b - 1, b, b + 1}
    return sorted(o for o in offs if 0 <= o and o + m <= n)


# ---- FASTA -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [5, 17, CAP])
@pytest.mark.parametrize("eol", [b"\n", b"\r\n"])
def test_fasta_planted_variants_uniform_and_streamed(tmp_path, m, eol):
    """uniform-line records (cut into pieces) and norm = 0 records longer than a piece (streamed window by window), each
    with one planted variant of 0 .. 4 substitutions at an offset around a piece boundary; the lines (61 bases) put
    line breaks inside every long pattern"""
    n = 2 * PIECE + CAP + 100
    pat = rand_seq(m, 7000 + m)
    offs = around_pieces(m, n) + [0, n - m, 30, 58]
    seqs = planted(n, pat, offs, 100 * m)
    recs = []
    for i, s in enumerate(seqs):
        if i % 3 == 2:                                                          # a blank line in the middle: norm = 0
            recs.append(b">n%d" % i + eol + wrap(s[:1000], 61, eol) + eol + wrap(s[1000:], 61, eol))
        else:
            recs.append(b">u%d" % i + eol + wrap(s, 61, eol))
    data = b"".join(recs)
    fa = pyfastx.Fasta(write(tmp_path, "v%d_%d.fa" % (m, len(eol)), data))
    rows, hays = S.whole_records(data)
    assert hays == seqs and 0 in rows["norm"].tolist() and 1 in rows["norm"].tolist()
    check(fa, hays, [pat])
    # every planted variant is found with its own count once k reaches it, and not before
    for k in ks(m):
        rid, start, minus, mm = fa.locate_approx(pat, k, "both")
        for i, o in enumerate(offs):
            d = i % 5 if i % 5 < m else 0
            sel = (rid == i) & (start == o) & (minus == bool(i & 1))
            assert int(sel.sum()) == (1 if d <= k else 0), (i, o, k)
            if d <= k:
                assert int(mm[sel][0]) == d


def test_fasta_uppercase_and_slices(tmp_path):
    seq = rand_seq(3 * PIECE + 500, 11, b"acgtACGTn")
    other = rand_seq(700, 12, b"acgt")
    data = b">a\n" + wrap(seq, 70) + b">b\n" + wrap(other, 50)
    fa = pyfastx.Fasta(write(tmp_path, "u.fa", data), uppercase=True)
    fl = pyfastx.Fasta(str(tmp_path / "u.fa"))
    _, up = S.whole_records(data, upper=True)
    _, low = S.whole_records(data)
    assert up[0] == seq.upper()
    pats = [seq[PIECE - 8:PIECE + 9].upper(), b"ACGTN", b"acgt", other[100:117].upper()]
    check(fa, up, pats, kset=(0, 2))
    check(fl, low, pats, kset=(0, 2))
    # slices through Engine.search_approx: (row_id, s, e), starts relative to s, nothing past e
    rows, _, _ = fxo.fasta_scan(data)
    eng, L = fa._st.engine, len(seq)
    pat = seq[PIECE - 10:PIECE + 7].upper()
    o = PIECE - 10
    qs = [(0, 0, L), (0, 0, o + 16), (0, 0, o + 17), (0, o, L), (0, 1, o + 17), (0, PIECE, L), (1, 3, 600), (0, 5, 5)]
    rid, s, e = (np.array(x, dtype=np.int64) for x in zip(*qs))
    hays = S.haystacks(data, rows, rid, s, e, upper=True)
    counts = A.strand_counts(hays, pat)
    for k in (0, 1, 3, 16):
        for _, mask in STRANDS:
            got = eng.search_approx(fa._st.dfile, fa._drows, rid, s, e, _cabi.X_UPPER, pat, k, mask)
            assert hit_list(got) == A.expected_from_counts(counts, k, mask), (k, mask)
    assert (0, o, 0, 0) in hit_list(eng.search_approx(fa._st.dfile, fa._drows, rid, s, e, _cabi.X_UPPER, pat, 0, 1))


# ---- FASTQ -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eol", [b"\n", b"\r\n"])
def test_fastq_read_lengths_and_planted_variants(tmp_path, eol):
    lengths = [0, 1, 4, 5, 16, 17, 150, 151, PIECE - 1, PIECE, PIECE + 1, 2 * PIECE + 3, 0, 150, 1, CAP, CAP + 40]
    seqs = [bytearray(rand_seq(n, 50 + i)) for i, n in enumerate(lengths)]
    pat = rand_seq(17, 4242)
    for i, s in enumerate(seqs):                                                # a variant at the start, middle, end
        if len(s) >= 17:
            for j, o in enumerate((0, len(s) // 2, len(s) - 17)):
                p = S.revcomp(pat) if (i + j) & 1 else pat
                s[o:o + 17] = variant(p, (i + j) % 5, 60 * i + j)
    seqs = [bytes(s) for s in seqs]
    data = b"".join(fq_record(b"r%d" % i, s, rand_seq(len(s), 900 + i), eol) for i, s in enumerate(seqs))
    fq = pyfastx.Fastq(write(tmp_path, "len%d.fq" % len(eol), data))
    _, hays = R.read_haystacks(data)
    assert hays == seqs
    check(fq, hays, [pat, pat[:5], "GATC", "T", seqs[11][PIECE - 600:PIECE + 424]])


def test_fastq_tiles_rounds_and_adjacent_long_reads(tmp_path):
    rng = np.random.default_rng(7)
    lens = [int(x) for x in rng.integers(100, 300, 200)]
    lens[40] = 3 * PIECE + 11
    lens[70] = lens[71] = 2 * PIECE + 1                                         # long reads next to each other
    lens[128:160] = [PIECE] * 32
    seqs = [rand_seq(n, 1000 + i) for i, n in enumerate(lens)]
    body = [fq_record(b"q%d" % i, s) for i, s in enumerate(seqs)]
    pats = [seqs[40][PIECE - 3:PIECE + 9], seqs[71][:12], seqs[70][-12:], seqs[150][-20:], b"GAATTC"]
    for count in (1, 31, 32, 33, 64, 65, 200):
        data = b"".join(body[:count])
        fq = pyfastx.Fastq(write(tmp_path, "t%d.fq" % count, data))
        _, hays = R.read_haystacks(data)
        check(fq, hays, pats, kset=(0, 2, 3))


def test_fastq_windows_never_run_past_a_read(tmp_path):
    """patterns that would be within k only by running into the '\\r', the '+' line, the quality line or the next read"""
    for eol in (b"\n", b"\r\n"):
        n = 40
        names = [rand_seq(10, 10 + i) for i in range(n)]
        seqs = [rand_seq(20 + (i % 7) * 31, 100 + i) for i in range(n)]
        quals = [rand_seq(len(s), 200 + i) for i, s in enumerate(seqs)]
        data = b"".join(fq_record(nm, s, q, eol) for nm, s, q in zip(names, seqs, quals))
        fq = pyfastx.Fastq(write(tmp_path, "b%d.fq" % len(eol), data))
        _, hays = R.read_haystacks(data)
        for i in range(n - 1):
            after = eol + b"+" + eol + quals[i] + eol + b"@" + names[i + 1]
            for a in (1, 3, 8):                                                 # bytes of the read the window keeps
                for b in (1, 2, 5):                                             # bytes it would take past the read's end
                    pat = seqs[i][-a:] + after[:b]
                    for k in sorted({b - 1, b, len(pat) - 1}):
                        if not 0 <= k < len(pat):
                            continue
                        exp = A.expected_hits(hays, pat, k, 3)
                        assert all(q != i or s < len(seqs[i]) - len(pat) + 1 for q, s, _, _ in exp)
                        if k < b:
                            assert (i, len(seqs[i]) - a, 0, 0) not in exp
                        got = approx_list(fq, pat, k, "both")
                        assert got == exp, (i, a, b, k)


def test_fastq_raw_bytes(tmp_path):
    lower = rand_seq(700, 3, b"acgtnACGTN")
    high = rand_seq(300, 5, b"ACGT\x80\xe9\xff")
    seqs = [b"TTAC GTAA", b"AC\tGTAC GT", lower, high, b"TTGAATTCAAGAATTCGGATCC" * 20, b"A" * 5000,
            b"AAAACAAAA" * 10, b"N" * 40 + b"ACGTACGTAC" + b"N" * 40]
    data = b"".join(fq_record(b"x%d" % i, s) for i, s in enumerate(seqs))
    fq = pyfastx.Fastq(write(tmp_path, "raw.fq", data))
    _, hays = R.read_haystacks(data)
    assert hays == seqs
    check(fq, hays, ["AC GT", "acgt", "GAATTC", "GGATCC", "ACGTACGTAC", "NNNNACGT", lower[100:130], high[10:25],
                     b"\xe9\x80\xff", "AAAA", "TTTTT", "CAG"])
    # on an A-run a pattern containing an A, with k = m - 1, hits at every start
    for pat in ("CAG", "AAAAAAT", "TTTTTTTTTTTTA"):
        rid, start, minus, mm = fq.locate_approx(pat, len(pat) - 1, "+")
        assert int((rid == 5).sum()) == 5000 - len(pat) + 1
        assert set(mm[rid == 5].tolist()) == {len(pat) - pat.count("A")}


# ---- both formats --------------------------------------------------------------------------------------------------------
def test_zero_mismatches_is_locate(tmp_path):
    fa = pyfastx.Fasta(write(tmp_path, "z.fa", synth.synth_fasta(50, seed=3)))
    fq = pyfastx.Fastq(write(tmp_path, "z.fq", synth.synth_fastq(400, seed=4)))
    for obj in (fa, fq):
        for pat in ("GAATTC", "ACG", "T", "ACGTTGCA"):
            for strand, _ in STRANDS:
                rid, start, minus = obj.locate(pat, strand)
                r2, s2, m2, mm = obj.locate_approx(pat, 0, strand)
                assert np.array_equal(rid, r2) and np.array_equal(start, s2) and np.array_equal(minus, m2)
                assert mm.dtype == np.int32 and not mm.any()


def _bgzf(data):
    L = _cabi.lib()
    a = np.frombuffer(data, np.uint8)
    out, n = C.c_void_p(), C.c_int64(0)
    _cabi.check(L.fxg_bgzf_compress_host(a.ctypes.data, a.size, 6, C.byref(out), C.byref(n)))
    comp = C.string_at(out.value, n.value)
    L.fxg_free_host(out)
    assert gzip.decompress(comp) == data
    return comp


@pytest.mark.parametrize("fmt", ["fa", "fq"])
def test_every_way_of_opening_gives_the_same_hits(tmp_path, fmt):
    data = synth.synth_fasta(60, seed=30) if fmt == "fa" else synth.synth_fastq(500, seed=31, read_len=151)
    cls = pyfastx.Fasta if fmt == "fa" else pyfastx.Fastq
    hays = S.whole_records(data)[1] if fmt == "fa" else R.read_haystacks(data)[1]
    plain = cls(write(tmp_path, "p." + fmt, data))
    again = cls(str(tmp_path / ("p." + fmt)))                                 # loads the .fxi written by the first open
    gz = cls(write(tmp_path, "p.%s.gz" % fmt, _bgzf(data)))
    assert gz.is_gzip and gz._st.bgzf_members > 1
    pat = hays[1][100:112]
    counts = A.strand_counts(hays, pat)
    for k in (0, 1, 2, 3, 11):
        exp = A.expected_from_counts(counts, k, 3)
        assert approx_list(plain, pat, k, "both") == exp
        assert approx_list(again, pat, k, "both") == exp
        assert approx_list(gz, pat, k, "both") == exp


def test_partial_and_empty_fastq(tmp_path):
    data = synth.synth_fastq(200, seed=33)
    part = data + b"@tail\nGAATTCGAATTC\n+\n"
    fq = pyfastx.Fastq(write(tmp_path, "part.fq", part))
    _, hays = R.read_haystacks(part)
    assert len(fq) == 200 == len(hays)
    check(fq, hays, ["GAATTCGAATTC"], kset=(0, 2))
    fq = pyfastx.Fastq(write(tmp_path, "none.fq", b"@only\nACGTACGT\n+\n"))
    assert len(fq) == 0
    rid, start, minus, mm = fq.locate_approx("ACGT", 1, "both")
    assert rid.size == start.size == minus.size == mm.size == 0
    assert (rid.dtype, start.dtype, minus.dtype, mm.dtype) == (np.int64, np.int64, bool, np.int32)


def test_arguments_and_reported_windows(tmp_path):
    fa = pyfastx.Fasta(write(tmp_path, "a.fa", synth.synth_fasta(20, seed=5)))
    fq = pyfastx.Fastq(write(tmp_path, "a.fq", synth.synth_fastq(300, seed=6)))
    for obj in (fa, fq):
        for bad in (1.0, "1", None, True, False, np.bool_(True)):
            with pytest.raises(TypeError):
                obj.locate_approx("ACGT", bad)
        for bad in (-1, 4, 5):
            with pytest.raises(ValueError):
                obj.locate_approx("ACGT", bad)
        for bad in ("", b"", "A" * (CAP + 1)):
            with pytest.raises(ValueError):
                obj.locate_approx(bad, 0)
        for bad in ("x", "+-", None):
            with pytest.raises(ValueError):
                obj.locate_approx("ACGT", 1, strand=bad)
        assert approx_list(obj, "GATCA", np.int64(1), "both") == approx_list(obj, b"GATCA", 1, "both")
        assert approx_list(obj, "GATCA", 1, "+") == approx_list(obj, bytearray(b"GATCA"), 1, "+")
    eng = fq._st.engine
    with pytest.raises(_cabi.FxgError):
        eng.search_reads_approx(fq._st.dfile, fq._drows, b"ACGT", 4, 1)
    with pytest.raises(_cabi.FxgError):
        eng.search_approx(fa._st.dfile, fa._drows, None, None, None, 0, b"ACGT", -1, 1)
    # every reported window, fetched through extraction / reads_many, has the reported count
    pat = b"ACGTTGCATG"
    rc = np.frombuffer(S.revcomp(pat), np.uint8)
    pw = np.frombuffer(pat, np.uint8)
    rid, start, minus, mm = fa.locate_approx(pat, 3, "both")
    assert rid.size > 0
    out, _, _ = fa._st.engine.extract(fa._st.dfile, fa._drows, rid, start, start + len(pat), np.zeros(rid.size, np.int32))
    win = out.reshape(-1, len(pat))
    assert np.array_equal((win != np.where(minus[:, None], rc, pw)).sum(axis=1), mm)
    rid, start, minus, mm = fq.locate_approx(pat, 3, "both")
    assert rid.size > 0
    seq, _, off = fq.reads_many(rid, want_qual=False)
    win = np.stack([seq[off[i] + start[i]:off[i] + start[i] + len(pat)] for i in range(rid.size)])
    assert np.array_equal((win != np.where(minus[:, None], rc, pw)).sum(axis=1), mm)


def test_random_draws(tmp_path):
    fdata = synth.synth_fasta(400, seed=20240601)
    qdata = synth.synth_fastq(3000, seed=20240602)
    fa = pyfastx.Fasta(write(tmp_path, "r.fa", fdata))
    fq = pyfastx.Fastq(write(tmp_path, "r.fq", qdata))
    fh, qh = S.whole_records(fdata)[1], R.read_haystacks(qdata)[1]
    rng = np.random.default_rng(99)
    for t in range(300):
        obj, hays = (fa, fh) if t & 1 else (fq, qh)
        kind = (t >> 1) % 3
        if kind < 2:
            h = hays[int(rng.integers(0, len(hays)))]
            a = int(rng.integers(0, len(h) - 40))
            pat = h[a:a + int(rng.integers(1, 41))]
            if kind == 1:
                pat = S.revcomp(pat)
        else:
            pat = rand_seq(int(rng.integers(8, 30)), 5000 + t)
        k = int(rng.integers(0, min(len(pat), 5)))
        strand, mask = STRANDS[(t // 6) % 3]
        assert approx_list(obj, pat, k, strand) == A.expected_hits(hays, pat, k, mask), (t, pat, k, strand)
