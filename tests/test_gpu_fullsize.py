"""BASELINE.json full sizes on one GPU, checked through size-independent properties (the oracle
would need minutes per case here): the C2 10 GB FASTA (1M records) and a C4-shaped FASTQ are generated
in HBM; expected rows follow analytically from the generator's layout; extraction is checked by
round trips (RC of RC is the identity, strands agree base by base) and against sampled oracle
answers on bytes downloaded from the same buffer."""
import numpy as np
import pytest

from oracle import fxo
from pyfastx_b200 import _cabi, engine, synth

pytestmark = pytest.mark.gpu
RC = _cabi.X_REVERSE | _cabi.X_COMPLEMENT


@pytest.fixture(scope="module")
def eng():
    return engine.get_engine(0)


def _ndig(v):
    return np.floor(np.log10(np.maximum(v, 1))).astype(np.int64) + 1


def test_c2_fasta_10gb_rows_and_extraction(eng):
    L = _cabi.lib()
    n = 1_000_000
    lengths = synth.fasta_lengths(n, 20240601)
    sizes = synth.fasta_record_sizes(lengths)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(sizes, out=off[1:])
    total = int(off[-1])
    assert 10.0e9 < total < 10.4e9
    f = eng.alloc_file(total)
    dl, do = eng.upload_rows(lengths), eng.upload_rows(off)
    _cabi.check(L.fxg_synth_fasta_dev(eng.ctx, 20240601, dl.devptr, do.devptr, n, 0, 80, f.devptr))
    eng.sync()
    rows, st, drows = eng.fasta_scan(f, keep_device_rows=True)
    # analytic rows from the generator layout
    idx = np.arange(1, n + 1, dtype=np.int64)
    hdr = len(b">seq synthetic len=") + _ndig(idx) + _ndig(lengths) + 1
    assert st["n_rows"] == n and st["total_len"] == int(lengths.sum()) and st["end_position"] == total
    assert np.array_equal(rows["boff"], off[:-1] + hdr)
    assert np.array_equal(rows["blen"], lengths + (lengths + 79) // 80)
    assert np.array_equal(rows["slen"], lengths)
    assert np.array_equal(rows["llen"], np.minimum(lengths, 80) + 1)
    assert (rows["elen"] == 1).all() and (rows["norm"] == 1).all()
    assert np.array_equal(rows["dlen"], hdr - 2) and np.array_equal(rows["nlen"], 3 + _ndig(idx))
    # 80-column lines, the last one no longer: every record has uniform lines (pad[0]), the other pad bytes stay 0
    assert (rows["pad"][:, 0] == 1).all() and (rows["pad"][:, 1:] == 0).all()
    # extraction round trips on 2M random windows of mixed length
    rid, s, e, minus = synth.random_queries(lengths, 2_000_000, seed=123, mixed=True)
    fl_plus = np.zeros(rid.size, dtype=np.int32)
    fl_rc = np.full(rid.size, RC, dtype=np.int32)
    a, off_a, acgt = eng.extract(f, drows, rid, s, e, fl_plus, want_acgt=True)
    b, off_b, _ = eng.extract(f, drows, rid, s, e, fl_rc)
    assert np.array_equal(off_a, off_b) and off_a[-1] == int((e - s).sum())
    assert np.isin(a, np.frombuffer(b"ACGT", np.uint8)).all()            # nothing but bases: newlines stripped
    assert np.array_equal(acgt.sum(axis=1), e - s)                       # fused counters see every base
    lut = fxo.complement_lut()
    # RC output, reversed per query, complemented again == forward output
    k = 20000
    for i in range(0, rid.size, rid.size // k):
        x = a[off_a[i]:off_a[i + 1]]
        y = b[off_b[i]:off_b[i + 1]]
        assert np.array_equal(lut[y][::-1], x)
    # sampled oracle answers computed from the bytes in HBM
    for i in range(0, rid.size, rid.size // 300):
        r = rows[rid[i]]
        rec0 = int(r["boff"])
        raw = f.download(rec0, int(r["blen"])).tobytes()
        local = np.zeros(1, dtype=fxo.FASTA_ROW)
        for fld in ("blen", "slen", "llen", "elen", "norm", "dlen", "nlen"):
            local[fld] = r[fld]
        local["boff"] = 0
        assert fxo.subseq(raw, local[0], int(s[i]), int(e[i])) == a[off_a[i]:off_a[i + 1]].tobytes()
        assert fxo.subseq(raw, local[0], int(s[i]), int(e[i]), fxo.REVERSE | fxo.COMPLEMENT) == b[off_b[i]:off_b[i + 1]].tobytes()
    # the generator's bases, independently: base k of record i is "ACGT"[mix(key) >> 62]
    for i in range(0, n, n // 50):
        got, _, _ = eng.extract(f, drows, [i], [0], [int(lengths[i])], [0])
        assert np.array_equal(got, synth.bases(20240601, i, int(lengths[i])))
    f.free()


def test_c4_fastq_shape_rows(eng):
    L = _cabi.lib()
    n = 12_000_000                                     # 3.9 GB, same record shape as the 40 GB C4 file
    fixed = 5 + 11 + 1 + 150 + 1 + 2 + 150 + 1
    idx = np.arange(1, n + 1, dtype=np.int64)
    rec = fixed + _ndig(idx)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(rec, out=off[1:])
    f = eng.alloc_file(int(off[-1]))
    _cabi.check(L.fxg_synth_fastq_dev(eng.ctx, 20240602, n, 0, 150, None, f.devptr))
    eng.sync()
    rows, st, drows = eng.fastq_scan(f, keep_device_rows=True)
    assert st["n_rows"] == n and st["n_lines"] == 4 * n and st["total_len"] == 150 * n
    hl = 5 + _ndig(idx) + 11                            # name line without the newline
    assert np.array_equal(rows["dlen"], hl) and np.array_equal(rows["nlen"], 4 + _ndig(idx))
    assert np.array_equal(rows["soff"], off[:-1] + hl + 1)
    assert np.array_equal(rows["qoff"], off[:-1] + hl + 1 + 150 + 1 + 2)
    assert (rows["rlen"] == 150).all()
    ids = np.random.default_rng(5).integers(0, n, size=500000)
    seq, qual, roff = eng.reads(f, drows, ids, rlens=rows["rlen"][ids])
    assert roff[-1] == 150 * ids.size
    assert np.isin(seq, np.frombuffer(b"ACGT", np.uint8)).all() and qual.min() >= 35 and qual.max() <= 70
    for j in range(0, ids.size, 5000):
        i = int(ids[j])
        assert np.array_equal(seq[roff[j]:roff[j + 1]], synth.bases(20240602, i, 150))
        assert np.array_equal(qual[roff[j]:roff[j + 1]], synth.quals(20240602, i, 150))
    f.free()
