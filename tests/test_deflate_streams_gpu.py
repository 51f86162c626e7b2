"""The GPU DEFLATE decoder on hand-built streams (tests/deflatelib.py), past the first round of member slots of
inflate_thread_kernel, and across hundreds of zran checkpoints of inflate_points_kernel: every verdict is zlib's,
every accepted byte is zlib's, and a rejected member writes nothing outside its own output slot."""
import ctypes as C
import gzip
import random

import numpy as np
import pytest

import deflatelib as D
from pyfastx_b200 import _cabi, synth

pytestmark = pytest.mark.gpu

CATALOGUE = D.catalogue()
SENTINEL = 0xA5
# member slots per SM in one round of inflate_thread_kernel: FXG_MT_WARPS (36, csrc/fxg_inflate.cu) warps of 32
# lanes, one member per lane; member m is decoded in round m // (sm_count * 1152) by the lane of slot m % that
MEMBERS_PER_SM = 36 * 32


@pytest.fixture(scope="module")
def eng():
    from pyfastx_b200 import engine
    return engine.get_engine(0)


def inflate_members(eng, members):
    """fxg_inflate_members_dev on members laid end to end, offsets in device tables; the output buffer is filled with
    a sentinel first and has 256 sentinel bytes past out_cap.  -> (status, output incl. the tail, uncompressed offsets)"""
    buf, co, uo = D.pack_members(members)
    n, total = len(members), uo[-1]
    f = eng.stage_bytes(buf)
    dco, duo = eng.upload_rows(np.array(co, np.int64)), eng.upload_rows(np.array(uo, np.int64))
    dout = eng.upload_rows(np.full(total + 256, SENTINEL, np.uint8))
    dst = eng.upload_rows(np.full(n, -1, np.int32))
    try:
        _cabi.check(_cabi.lib().fxg_inflate_members_dev(eng.ctx, f.handle, dco.devptr, duo.devptr, n, dout.devptr, total,
                                                        dst.devptr))
        eng.sync()
        st = np.zeros(n, np.int32)
        out = np.zeros(total + 256, np.uint8)
        _cabi.check(_cabi.lib().fxg_rows_download(eng.ctx, dst.devptr, n, 4, st.ctypes.data))
        _cabi.check(_cabi.lib().fxg_rows_download(eng.ctx, dout.devptr, total + 256, 1, out.ctypes.data))
    finally:
        for d in (dco, duo, dout, dst):
            d.free()
        f.free()
    return st, out, np.array(uo, np.int64)


# ---- (a) the catalogue in one BGZF file ------------------------------------------------------------------------------
@pytest.mark.parametrize("crc", ["on", "off"])
def test_catalogue_in_one_file(eng, monkeypatch, crc):
    """status zero exactly where zlib accepts (the decoder's own rejection path where the catalogue names one, with
    or without the CRC kernel), byte-exact output, and no byte written outside a rejected member's slot"""
    if crc == "off":
        monkeypatch.setenv("FXG_BGZF_CRC", "0")
    st, out, uo = inflate_members(eng, [s.member() for s in CATALOGUE] + [D.BGZF_EOF])
    for i, s in enumerate(CATALOGUE):
        if s.out is None:
            assert st[i] != 0 and (s.status is None or st[i] == s.status), (s.name, st[i])
        else:
            assert st[i] == 0, (s.name, st[i])
            assert out[uo[i]:uo[i + 1]].tobytes() == s.out, s.name
    assert st[-1] == 0 and (out[uo[-1]:] == SENTINEL).all()


@pytest.mark.parametrize("crc", ["on", "off"])
def test_stage_bgzf_rejects_every_member_zlib_rejects(eng, monkeypatch, crc):
    """a BGZF file holding one rejected member between valid ones does not open -- with the CRC check off too: each
    rejection comes from the decoder, not from the CRC-32; the valid entries together open byte-exact"""
    if crc == "off":
        monkeypatch.setenv("FXG_BGZF_CRC", "0")
    nb = next(s for s in CATALOGUE if s.name == "fixed_only")
    for s in CATALOGUE:
        if s.out is None:
            z = nb.member() + s.member() + nb.member() + D.BGZF_EOF
            with pytest.raises(_cabi.FxgError, match="member 1 is corrupt"):
                eng.stage_bgzf(np.frombuffer(z, np.uint8))
    ok = [s for s in CATALOGUE if s.out is not None and len(s.member()) <= 65536]     # BSIZE is 16 bits
    assert len(ok) >= len([s for s in CATALOGUE if s.out is not None]) - 1
    f = eng.stage_bgzf(np.frombuffer(b"".join(s.member() for s in ok) + D.BGZF_EOF, np.uint8))
    assert f.n_members == len(ok) + 1 and f.download().tobytes() == b"".join(s.out for s in ok)
    f.free()


# ---- (b) past the first round of member slots --------------------------------------------------------------------
def random_member(rng, k):
    """a valid member of 0 to a few hundred bytes: stored, fixed, dynamic or a mix, literals and matches"""
    w = D.Writer()
    kinds = [("stored",), ("fixed",), ("dynamic",), ("fixed", "stored", "dynamic")][k % 4]
    for j, kind in enumerate(kinds):
        last = j == len(kinds) - 1
        n = rng.randrange(0, 60)
        if kind == "stored":
            w.stored(bytes(rng.choice(b"ACGTN\n") for _ in range(n)), last=last)
            continue
        syms, have = [], len(w.data)
        while len(syms) < n:
            if have and rng.random() < 0.3:
                m = D.Match(258 if rng.random() < 0.02 else rng.randrange(3, 20), rng.randrange(1, have + 1))
                syms.append(m)
                have += m.length
            else:
                syms.append(rng.choice(b"ACGTacgt@+\n"))
                have += 1
        (w.fixed if kind == "fixed" else w.dynamic)(syms, last=last)
    return D.gzip_member(w.getvalue(), bytes(w.data)), bytes(w.data)


def test_members_past_the_first_round(eng):
    """at least 2.5 rounds of member slots, rejected members at the last slot of a round, the first slot of the next
    and elsewhere in rounds two and three: every status and every byte against zlib, and hundreds of thousands of
    short, unaligned ranges through the CRC kernel"""
    R = eng.sm_count * MEMBERS_PER_SM
    n = 5 * R // 2 + 1234
    rng = random.Random(11)
    pool = [random_member(rng, k) for k in range(800)]
    for m, data in pool:
        assert gzip.decompress(m) == data                    # zlib's verdict on every pool member
    bad = [s for s in CATALOGUE if s.out is None]
    bad_at = sorted({R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1, n - 1} | set(rng.sample(range(R, n), 60)))
    pick = [rng.randrange(len(pool)) for _ in range(n)]
    members, want = [], []
    bad_of = dict(zip(bad_at, (bad[i % len(bad)] for i in range(len(bad_at)))))
    for i in range(n):
        if i in bad_of:
            members.append(bad_of[i].member())
            want.append(None)
        else:
            members.append(pool[pick[i]][0])
            want.append(pool[pick[i]][1])
    st, out, uo = inflate_members(eng, members)
    assert sorted(np.flatnonzero(st).tolist()) == bad_at
    for i, s in bad_of.items():
        assert s.status is None or st[i] == s.status, (i, s.name, st[i])
    valid = np.array([w is not None for w in want])
    mask = np.repeat(valid, np.diff(uo))
    exp = np.frombuffer(b"".join(w if w is not None else bytes(int(uo[i + 1] - uo[i])) for i, w in enumerate(want)), np.uint8)
    got = out[:uo[-1]]
    assert np.array_equal(got[mask], exp[mask])
    assert (out[uo[-1]:] == SENTINEL).all()


# ---- (c) many checkpoints -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def fastq16():
    raw = synth.synth_fastq(52000, seed=5)
    assert len(raw) >= 16 << 20
    return raw


def stage_points(eng, z, gz):
    a = np.frombuffer(z, dtype=np.uint8)
    h = C.c_void_p()
    _cabi.check(_cabi.lib().fxg_file_from_gzip_points_host(eng.ctx, a.ctypes.data, a.size, C.byref(gz), C.byref(h)))
    from pyfastx_b200.engine import DeviceFile
    return DeviceFile(eng, h)


def test_hundreds_of_checkpoints(eng, fastq16):
    """plain gzip at levels 0, 1, 6 and 9, checkpoints every 32 KiB: several hundred segments per file (several CTAs),
    every bit offset 0..7 among them, and the output equals the input"""
    from test_gzip_cpu import inflate_host
    bits = set()
    for level in (0, 1, 6, 9):
        z = gzip.compress(fastq16, compresslevel=level, mtime=0)
        got, gz, pts, h = inflate_host(z, 32768)
        try:
            assert got == fastq16
            assert gz.npoints >= 240 and (gz.npoints + 63) // 64 >= 4, (level, gz.npoints)
            bits |= set(pts["bits"].tolist())
            f = stage_points(eng, z, gz)
            assert f.size == len(fastq16) and f.download().tobytes() == fastq16
            f.free()
        finally:
            _cabi.lib().fxg_gzip_free(h)
    assert bits == set(range(8))


def test_window_edge_on_the_gpu(eng):
    """the segment that starts at the window-edge checkpoint decodes on the GPU; a changed window byte that its first
    match reads makes the combined CRC-32 differ from the trailer's"""
    from test_gzip_cpu import inflate_host
    s = next(s for s in CATALOGUE if s.name == "window_edge")
    z = s.member(bgzf=False)
    got, gz, pts, h = inflate_host(z, 32768)
    try:
        assert pts["ucmp"].tolist() == [0, 40000]
        f = stage_points(eng, z, gz)
        assert f.download().tobytes() == s.out
        f.free()
        C.c_uint8.from_address(gz.windows).value ^= 0xff      # window byte 0 of checkpoint 1
        with pytest.raises(_cabi.FxgError, match="CRC-32") as ei:
            stage_points(eng, z, gz)
        assert ei.value.code == _cabi.FXG_EFORMAT
    finally:
        _cabi.lib().fxg_gzip_free(h)


def test_empty_inputs_stage_to_size_zero(eng):
    """an empty plain gzip (one checkpoint, no output) and a BGZF file of just the EOF member"""
    from test_gzip_cpu import inflate_host
    z = gzip.compress(b"", mtime=0)
    got, gz, pts, h = inflate_host(z, 32768)
    try:
        assert got == b"" and gz.npoints == 1
        f = stage_points(eng, z, gz)
        assert f.size == 0
        f.free()
    finally:
        _cabi.lib().fxg_gzip_free(h)
    f = eng.stage_bgzf(np.frombuffer(D.BGZF_EOF, np.uint8))
    assert f.size == 0 and f.n_members == 1
    f.free()
