"""Hand-built DEFLATE streams (tests/deflatelib.py) against zlib and against the host build of the decoder the GPU
runs (pyfastx_b200/csrc/fxg_inflate_core.cuh): every valid shape decodes byte-exact, every stream zlib rejects is
rejected, and a rejected member writes nothing outside its own output slot."""
import ctypes as C
import gzip
import os
import subprocess
import zlib

import numpy as np
import pytest

import deflatelib as D

HERE = os.path.dirname(os.path.abspath(__file__))
CATALOGUE = D.catalogue()
SENTINEL = 0xA5

# zlib's message for every stream it rejects: each entry fails for the reason its name gives
ZLIB_ERROR = {
    "btype_3": "invalid block type",
    "stored_nlen_mismatch": "invalid stored block lengths",
    "hlit_287": "too many length or distance symbols",
    "hdist_31": "too many length or distance symbols",
    "repeat_16_first": "invalid bit length repeat",
    "repeat_past_hlit_hdist": "invalid bit length repeat",
    "missing_eob": "incorrect data check",                 # zlib decodes on into the trailer
    "lit_code_oversubscribed": "invalid literal/lengths set",
    "dist_code_oversubscribed": "invalid distances set",
    "lit_code_incomplete": "invalid literal/lengths set",
    "dist_code_incomplete": "invalid distances set",
    "cl_code_oversubscribed": "invalid code lengths set",
    "cl_code_incomplete": "invalid code lengths set",
    "junk_before_trailer": "incorrect data check",
    "junk_after_stored": "incorrect data check",
    "fixed_lit_286": "invalid literal/length code",
    "fixed_lit_287": "invalid literal/length code",
    "fixed_dist_30": "invalid distance code",
    "fixed_dist_31": "invalid distance code",
    "dist_past_member_start": "invalid distance too far back",
    "output_longer_than_isize": "incorrect length check",
    "output_shorter_than_isize": "incorrect length check",
    "truncated_stored": "incomplete or truncated stream",
    "truncated_dynamic": "incomplete or truncated stream",
}


def by_name(name):
    return next(s for s in CATALOGUE if s.name == name)


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("deflate_streams") / "inflate_core_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++",
                           os.path.join(HERE, "native", "inflate_core_host.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.fxi_host_inflate.restype = C.c_int
    lib.fxi_host_inflate.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    lib.fxi_host_inflate_points.restype = C.c_int
    lib.fxi_host_inflate_points.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    return lib


def test_catalogue_names_every_rejection():
    names = [s.name for s in CATALOGUE]
    assert len(set(names)) == len(names)
    assert {s.name for s in CATALOGUE if s.out is None} == set(ZLIB_ERROR)
    assert sum(s.out is not None for s in CATALOGUE) >= 30


@pytest.mark.parametrize("name", [s.name for s in CATALOGUE])
def test_catalogue_is_zlibs_verdict(name):
    """the expected answer of every entry is zlib's: the bytes of its gzip member (wbits=31: header, data, CRC-32 and
    ISIZE checked), or zlib's error for the reason the entry is named after"""
    s = by_name(name)
    if s.out is None:
        with pytest.raises(zlib.error, match=ZLIB_ERROR[name].replace("/", ".")):
            zlib.decompress(s.member(bgzf=False), 31)
        assert D.zlib_verdict(s) is None
        return
    assert D.zlib_verdict(s) == s.out
    assert zlib.decompress(s.deflate, -15) == s.out                # the raw deflate data alone
    d = zlib.decompressobj(31)                                      # the BGZF form: extra subfields, then 'BC'
    assert d.decompress(s.member()) == s.out and d.eof and not d.unused_data


def host_inflate(core, members):
    """members decoded by the host build, as the kernel lays them out; the output buffer is filled with a sentinel
    first and has 64 sentinel bytes past out_cap"""
    buf, co, uo = D.pack_members(members)
    a = np.frombuffer(buf, dtype=np.uint8).copy()
    co, uo = np.array(co, np.int64), np.array(uo, np.int64)
    out = np.full(int(uo[-1]) + 64, SENTINEL, dtype=np.uint8)
    st = np.full(len(members), -1, dtype=np.int32)
    core.fxi_host_inflate(a.ctypes.data, a.size, co.ctypes.data, uo.ctypes.data, len(members), out.ctypes.data, int(uo[-1]),
                          st.ctypes.data)
    return st, out, uo


@pytest.mark.parametrize("name", [s.name for s in CATALOGUE])
def test_host_decoder_gives_zlibs_verdict(core, name):
    """the entry between two valid members: status 0 exactly where zlib accepts, the bytes zlib gives, the decoder's
    rejection path for a rejected entry, and the neighbours' slots and the bytes past out_cap untouched"""
    s, nb = by_name(name), by_name("fixed_only")
    st, out, uo = host_inflate(core, [nb.member(), s.member(), nb.member()])
    assert st[0] == 0 and st[2] == 0
    if s.out is None:
        assert st[1] != 0
        if s.status is not None:
            assert st[1] == s.status
    else:
        assert st[1] == 0
        assert out[uo[1]:uo[2]].tobytes() == s.out
    assert out[uo[0]:uo[1]].tobytes() == nb.out and out[uo[2]:uo[3]].tobytes() == nb.out
    assert (out[uo[3]:] == SENTINEL).all()


def test_host_decoder_whole_catalogue_in_one_call(core):
    """every entry in one file, one call: per member the verdict and bytes do not depend on what came before"""
    st, out, uo = host_inflate(core, [s.member() for s in CATALOGUE])
    for i, s in enumerate(CATALOGUE):
        assert (st[i] == 0) == (s.out is not None), s.name
        if s.out is not None:
            assert out[uo[i]:uo[i + 1]].tobytes() == s.out, s.name
    assert (out[uo[-1]:] == SENTINEL).all()


def test_checkpoint_at_the_window_edge(core):
    """40,000 stored bytes, then a block that opens with a match at distance 32,768: with 32 KiB spacing the host pass
    puts a checkpoint at that block, and the segment decoded from it reads byte 0 of the checkpoint's window -- a
    different byte 0 changes exactly the first output byte of the segment"""
    from test_gzip_cpu import inflate_host
    from pyfastx_b200 import _cabi
    s = by_name("window_edge")
    z = s.member(bgzf=False)
    got, gz, pts, h = inflate_host(z, 32768)
    try:
        assert got == s.out and gzip.decompress(z) == s.out
        assert pts["ucmp"].tolist() == [0, 40000] and pts["has"].tolist() == [0, 1]
        assert pts["bits"][1] == 0                           # a stored block ends on a byte boundary
        win = np.frombuffer(pts["win"], dtype=np.uint8).copy()
        assert win.tobytes() == s.out[40000 - 32768:40000]
        a = np.frombuffer(z, dtype=np.uint8).copy()
        ucmp = np.array([0, 40000, len(s.out)], dtype=np.int64)

        def segments(window):
            out = np.zeros(len(s.out) + 64, dtype=np.uint8)
            st = np.full(2, -1, dtype=np.int32)
            core.fxi_host_inflate_points(a.ctypes.data, a.size, 2, pts["cmp"].ctypes.data, pts["bits"].ctypes.data,
                                         ucmp.ctypes.data, pts["has"].ctypes.data, window.ctypes.data, 32768,
                                         out.ctypes.data, len(s.out), st.ctypes.data)
            return st, out[:len(s.out)].tobytes()

        st, out = segments(win)
        assert st.tolist() == [0, 0] and out == s.out
        bad = win.copy()
        bad[0] ^= 0xff
        st, out = segments(bad)
        assert st.tolist() == [0, 0]
        diff = [i for i in range(len(s.out)) if out[i] != s.out[i]]
        assert diff == [40000]                             # only the match's first byte, window byte 0
    finally:
        _cabi.lib().fxg_gzip_free(h)
