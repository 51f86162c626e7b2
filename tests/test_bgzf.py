"""K6: BGZF inputs.  The member walk is host code (CPU test); the member-parallel inflate and the
Fasta/Fastq path on top of it run on the GPU and must reproduce zlib's output / the plain-file index
bit for bit (BASELINE.json configs[4] at test size)."""
import ctypes as C
import gzip
import os
import struct
import zlib

import numpy as np
import pytest

import gen
import goldenlib as G
from pyfastx_b200 import _cabi, synth


def bgzf_compress(data, level=6, block=0xff00):
    """BGZF writer (SAM spec 4.1): gzip members with a 'BC' extra field + the empty EOF member."""
    out = []
    for a in list(range(0, len(data), block)) + [None]:
        chunk = b"" if a is None else data[a:a + block]
        co = zlib.compressobj(level, zlib.DEFLATED, -15)
        comp = co.compress(chunk) + co.flush()
        bsize = len(comp) + 25
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize)
                   + comp + struct.pack("<II", zlib.crc32(chunk), len(chunk)))
    return b"".join(out)


def members(buf):
    lib = _cabi.lib()
    a = np.frombuffer(buf, dtype=np.uint8)
    n, tot = C.c_int64(0), C.c_int64(0)
    rc = lib.fxg_bgzf_members_host(a.ctypes.data, a.size, None, None, 0, C.byref(n), C.byref(tot))
    if rc:
        return rc, None, None, 0
    co = np.zeros(n.value + 1, dtype=np.int64)
    uo = np.zeros(n.value + 1, dtype=np.int64)
    rc = lib.fxg_bgzf_members_host(a.ctypes.data, a.size, co.ctypes.data, uo.ctypes.data, n.value + 1, C.byref(n), C.byref(tot))
    return rc, co, uo, tot.value


def test_member_table_host():
    data = synth.synth_fasta(30, seed=3)
    z = bgzf_compress(data)
    assert gzip.decompress(z) == data                      # a valid multi-member gzip stream
    rc, co, uo, tot = members(z)
    assert rc == 0 and tot == len(data)
    assert co[0] == 0 and co[-1] == len(z) and (np.diff(co) > 0).all()
    assert uo[-1] == len(data) and (np.diff(uo)[:-2] == 0xff00).all()      # full members, a partial one, EOF
    assert np.diff(uo)[-1] == 0                            # the EOF member is empty
    rc, *_ = members(gzip.compress(data))                  # plain gzip is not BGZF
    assert rc == _cabi.FXG_EFORMAT
    rc, *_ = members(z[:-10])
    assert rc == _cabi.FXG_EFORMAT


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["dna", "text", "stored", "tiny", "fastq", "binary"])
def test_gpu_inflate_matches_zlib(kind):
    from pyfastx_b200 import engine
    eng = engine.get_engine(0)
    rng = np.random.default_rng(7)
    if kind == "dna":
        data, level, block = synth.synth_fasta(400, seed=11), 6, 0xff00
    elif kind == "text":
        data, level, block = (b"the quick brown fox jumps over the lazy dog. " * 40000)[:1_500_000], 9, 0xff00
    elif kind == "stored":
        data, level, block = rng.integers(0, 256, size=300_000, dtype=np.uint8).tobytes(), 0, 0xff00
    elif kind == "tiny":
        data, level, block = synth.synth_fastq(60, seed=2), 6, 97          # many tiny members (fixed Huffman blocks)
    elif kind == "fastq":
        data, level, block = synth.synth_fastq(20000, seed=20240602), 1, 0xff00
    else:
        data, level, block = rng.integers(0, 256, size=500_000, dtype=np.uint8).tobytes(), 6, 30000
    z = bgzf_compress(data, level, block)
    f = eng.stage_bgzf(np.frombuffer(z, dtype=np.uint8))
    assert f.size == len(data)
    assert f.download().tobytes() == data
    f.free()


@pytest.mark.gpu
def test_corrupt_member_is_reported():
    from pyfastx_b200 import engine
    eng = engine.get_engine(0)
    z = bytearray(bgzf_compress(synth.synth_fasta(50, seed=5)))
    z[200] ^= 0xff                                           # inside the first member's deflate data
    with pytest.raises(_cabi.FxgError):
        eng.stage_bgzf(np.frombuffer(bytes(z), dtype=np.uint8))


@pytest.mark.gpu
def test_crc_mismatch_is_reported(monkeypatch):
    """a member that inflates to the right length but whose bytes differ from what the trailer's CRC-32 covers (here: the
    trailer's CRC field is altered; the deflate data is intact) is rejected like zlib rejects it -- and accepted with the
    check switched off, which proves that it is the CRC kernel that caught it"""
    from pyfastx_b200 import engine
    eng = engine.get_engine(0)
    data = synth.synth_fasta(50, seed=6)
    z = bytearray(bgzf_compress(data))
    rc, co, uo, tot = members(bytes(z))
    z[int(co[1]) - 8] ^= 0x01                                # first member's CRC32 field
    with pytest.raises(_cabi.FxgError) as ei:
        eng.stage_bgzf(np.frombuffer(bytes(z), dtype=np.uint8))
    assert "CRC-32" in str(ei.value)
    monkeypatch.setenv("FXG_BGZF_CRC", "0")
    f = eng.stage_bgzf(np.frombuffer(bytes(z), dtype=np.uint8))
    assert bytes(f.download()) == data
    f.free()


@pytest.mark.gpu
def test_fasta_on_bgzf_equals_plain(tmp_path):
    import pyfastx_b200 as pyfastx
    data = synth.synth_fasta(300, seed=20240601)
    plain = tmp_path / "p.fa"
    plain.write_bytes(data)
    bg = tmp_path / "b.fa.gz"
    bg.write_bytes(bgzf_compress(data))
    fa, fb = pyfastx.Fasta(str(plain)), pyfastx.Fasta(str(bg))
    assert fb.is_gzip and fb._st.bgzf_members > 1 and not fa.is_gzip
    assert fa.keys() == fb.keys() and len(fa) == 300
    for fld in ("boff", "blen", "slen", "llen", "dlen", "nlen", "elen", "norm"):
        assert np.array_equal(fa._rows[fld], fb._rows[fld])
    rid, s, e, minus = synth.random_queries(fa._rows["slen"], 3000, seed=124)
    a, oa, _ = fa.extract(rid, s, e, minus)
    b, ob, _ = fb.extract(rid, s, e, minus)
    assert np.array_equal(oa, ob) and np.array_equal(a, b)
    assert fb["seq7"][100:160].antisense == fa["seq7"][100:160].antisense
    # reference fixture through BGZF: same rows as the golden CRLF case
    case = [c for c in G.cases("fasta") if c["name"] == "test_fa_crlf"][0]
    raw = G.case_data(case)
    p2 = tmp_path / "t.fa.gz"
    p2.write_bytes(bgzf_compress(raw, block=4000))
    ft = pyfastx.Fasta(str(p2))
    q = case["queries"][3]
    assert ft[q["row"]][q["s"]:q["e"]].seq == q["seq"] and len(ft) == len(case["rows"])


@pytest.mark.gpu
def test_fastq_on_bgzf(tmp_path):
    import pyfastx_b200 as pyfastx
    data = gen.random_fastq(31, n_reads=4000)
    p = tmp_path / "r.fq.gz"
    p.write_bytes(bgzf_compress(data, level=4))
    q = tmp_path / "r.fq"
    q.write_bytes(data)
    fz, fp = pyfastx.Fastq(str(p)), pyfastx.Fastq(str(q))
    assert len(fz) == len(fp) == 4000 and fz.size == fp.size
    for i in (0, 1, 1234, 3999):
        assert (fz[i].seq, fz[i].qual, fz[i].name) == (fp[i].seq, fp[i].qual, fp[i].name)
