"""The sharded build's layouts and split points, without a GPU: every layout of tests/shardlib.py puts its cuts where
it says, and fxg_split_point_path (pread in 1 MiB windows) finds what shard.split_point_bytes finds on the same bytes,
with a window edge between a '\\n' and the '>' after it, inside a 3 MiB line, and at the ends of the file."""
import ctypes as C
import os

import pytest

import shardlib as S
from pyfastx_b200 import _cabi, shard


@pytest.fixture(scope="module")
def tmpdir_mod(tmp_path_factory):
    return str(tmp_path_factory.mktemp("shard_scale_cpu"))


def split_point_path(path, start, want_header):
    pos, size = C.c_int64(-1), C.c_int64(-1)
    _cabi.check(_cabi.lib().fxg_split_point_path(os.fsencode(path), int(start), 1 if want_header else 0,
                                                 C.byref(pos), C.byref(size)))
    assert size.value == os.path.getsize(path)
    return pos.value


@pytest.mark.parametrize("name", S.layout_ids())
def test_layout_aims(name):
    lay = S.layout(name)
    pts = lay.pts
    assert pts == sorted(pts) and pts[-1] == len(lay.data)
    for r in range(1, len(pts) - 1):                     # every cut is a place a split point could land
        p = pts[r]
        if p < len(lay.data):
            assert lay.data[p - 1:p] == b"\n", (name, r)
            if lay.mode == 0:
                assert lay.data[p:p + 1] == b">", (name, r)
    assert lay.aims
    for aim in lay.aims:
        assert S.check_aim(lay, aim), (name, aim)


def test_layouts_cover_the_issue_edges():
    """the layouts together reach every edge the GPU tests rely on"""
    ids = S.layout_ids()
    aims = [(S.layout(i), a) for i in ids for a in S.layout(i).aims]
    fq = [(lay, a) for lay, a in aims if lay.mode == 1]
    for p in range(4):
        for crlf in (False, True):
            assert any(a[0] == "phase" and a[2] == p and (("crlf",) in lay.aims) == crlf for lay, a in fq), (p, crlf)
    nl_bytes = {a[3] for _, a in fq if a[0] == "nl" and a[2] == 0}
    assert {2047, 2048} <= nl_bytes                                 # a shard's first newline at byte 2047 / 2048
    assert any(a[3] // S.REGION == S.EDGE_GROUP - 1 for _, a in fq if a[0] == "nl")    # ... in region 31
    assert max(a[2] for _, a in fq if a[0] == "edge_regions") > 2 * S.EDGE_GROUP    # edge lines past 64 regions
    assert any(a[0] == "no_eol_end" and a[1].endswith(b"\r") for _, a in fq)
    assert any(a[0] == "lines" and a[2] == 1 for _, a in fq) and any(a[0] == "lines" and a[2] == 2 for _, a in fq)
    kinds = {(lay.mode, a[0]) for lay, a in aims}
    for mode in (0, 1):
        for k in ("empty", "record_over_block", "blocks", "crlf"):
            assert (mode, k) in kinds, (mode, k)
    assert (0, "lead") in kinds and (0, "general") in kinds
    assert any(S.layout(i).full_name for i in ids)
    big = [S.layout(i) for i in ids if i.startswith("blocks_layout")]
    assert all(40e6 <= len(lay.data) <= 80e6 for lay in big) and len(big) == 2


@pytest.mark.parametrize("name", S.layout_ids())
def test_split_points_path_equal_bytes(name, tmpdir_mod):
    """all world + 1 split points from the file on disk equal those from the bytes, for worlds 1..16"""
    lay = S.layout(name)
    path = lay.write(tmpdir_mod)
    for world in range(1, 17):
        want = shard.split_points_bytes(lay.data, world, lay.mode == 0)
        assert shard.split_points_path(path, world, lay.mode == 0) == want, (name, world)


def test_split_point_path_window_edges(tmpdir_mod):
    """'\\n' as the last byte of a 1 MiB pread window with the '>' first in the next; a 3 MiB line without a newline;
    from = 0, 1, n - 1, n, n + 5"""
    data, x = S.split_window_file()
    assert data[x:x + 2] == b"\n>" and data.find(b"\n>") == x
    path = os.path.join(tmpdir_mod, "windows.fa")
    with open(path, "wb") as f:
        f.write(data)
    n = len(data)
    y = data.find(b"\n", x + 2)                          # end of the second header line
    z = data.find(b"\n", y + 1)                          # end of the 3 MiB line
    assert z - y - 1 == 3 * S.MiB and data[z + 1:z + 2] == b">"
    froms = S.split_froms(x, n) + S.split_froms(z, n) + [y + 2, y + 3, z, z + 1, z + 2]
    for k in (1, 2, 3):                                  # from inside the long line, windows ending on its bytes
        froms += [y + 2 + k * S.PREAD_WINDOW + d for d in (-1, 0, 1)]
    hits = set()
    for start in sorted(set(froms)):
        for hdr in (True, False):
            want = shard.split_point_bytes(data, start, hdr)
            assert split_point_path(path, start, hdr) == want, (start, hdr)
            hits.add(want)
    assert {x + 1, z + 1, n} <= hits


def test_split_point_path_no_header(tmpdir_mod):
    """a file without a header line: every header search returns n, line searches the next line start"""
    data = b"ACGTACGT\n" * 300000 + b"TTTT"                # 2.7 MB, unterminated last line
    path = os.path.join(tmpdir_mod, "noheader.txt")
    with open(path, "wb") as f:
        f.write(data)
    n = len(data)
    for start in [0, 1, 2, 8, 9, 10, S.PREAD_WINDOW - 1, S.PREAD_WINDOW, S.PREAD_WINDOW + 1, 2 * S.PREAD_WINDOW + 3,
                  n - 5, n - 4, n - 1, n, n + 5]:
        assert split_point_path(path, start, True) == n == shard.split_point_bytes(data, start, True), start
        assert split_point_path(path, start, False) == shard.split_point_bytes(data, start, False), start
