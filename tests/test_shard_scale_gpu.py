"""The sharded index build at real shard sizes, on one GPU: stage_path_range through its pinned-piece ring, the
one-rank C-ABI (fxg_scan_sharded with no communicator, fxg_shard_exchange with none), the split-phase scan of N
ranks run loop-back on the layouts of tests/shardlib.py (FASTQ shards starting inside 70-131 kB reads on every line
phase, LF and CRLF; shards of one line; empty shards; records longer than a prefix block; shards of several prefix
blocks), split_point_dev around its 4096-byte steps, and shard.build_index_sharded against the .fxi that
Fasta / Fastq write.  Every expected value comes from the whole-file oracle or plain Python on the bytes."""
import ctypes as C
import functools
import os

import numpy as np
import pytest

import shardlib as S
from oracle import fxo
from pyfastx_b200 import _cabi, engine, fxi, shard

pytestmark = pytest.mark.gpu

WORLDS = (2, 3, 5, 8, 16)
BIG_BASE = 1 << 33                                       # base offsets past 2^32


@pytest.fixture(scope="module")
def engs():
    es = [engine.Engine(0) for _ in range(max(WORLDS))]
    yield es
    for e in es:
        e.close()


@pytest.fixture(scope="module")
def stager():
    """stages every rank's range: one pinned ring (512 MiB) serves all emulated ranks"""
    e = engine.Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def tmpd(tmp_path_factory):
    return str(tmp_path_factory.mktemp("shard_scale_gpu"))


def assert_rows_equal(got, exp, what=""):
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    for f in exp.dtype.names:
        bad = np.nonzero(got[f] != exp[f])[0]
        assert bad.size == 0, "%s: field %s differs at rows %s: got %s expected %s" % (
            what, f, bad[:5], got[f][bad[:5]], exp[f][bad[:5]])


@functools.lru_cache(maxsize=None)
def expected(name):
    """whole-file oracle: (rows, total, n_lines or None, names)"""
    lay = S.layout(name)
    if lay.mode == 0:
        rows, total, _ = fxo.fasta_scan(lay.data, lay.full_name)
        return rows, total, None, fxo.fasta_names(lay.data, rows)
    rows, total, nl = fxo.fastq_scan(lay.data)
    return rows, total, nl, fxo.fastq_names(lay.data, rows)


OFFSET_FIELDS = {0: ("boff",), 1: ("soff", "qoff")}


# ---- 1. stage_path_range --------------------------------------------------------------------------------
def write_positional(path, n):
    """bytes that depend on their position (no two 16 MiB pieces alike)"""
    with open(path, "wb") as f:
        for o in range(0, n, S.RING_PIECE):
            i = np.arange(o, min(n, o + S.RING_PIECE), dtype=np.uint64)
            with np.errstate(over="ignore"):
                f.write(((i * np.uint64(2654435761)) >> np.uint64(13) ^ (i >> np.uint64(24))).astype(np.uint8).tobytes())


def check_staged(stager, path, mm, begin, end):
    f = stager.stage_path_range(path, begin, end)
    try:
        stop = len(mm) if end < 0 else min(end, len(mm))
        want = mm[begin:max(begin, stop)]
        assert f.size == want.size, (begin, end)
        got = f.download()
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (begin, end, bad[:5])
    finally:
        f.free()


def test_stage_path_range_piece_edges(stager, tmpd):
    """begin in {0, 1, 15, 16 MiB - 1, 16 MiB, 16 MiB + 1}, end in {begin, begin + 1, a piece edge +- 1, the end}"""
    P = S.RING_PIECE
    path = os.path.join(tmpd, "pieces.bin")
    n = 3 * P + 12345
    write_positional(path, n)
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    for begin in (0, 1, 15, P - 1, P, P + 1):
        for end in (begin, begin + 1, begin + P - 1, begin + P, begin + P + 1, begin + 2 * P + 1, -1):
            check_staged(stager, path, mm, begin, end)
    del mm


def test_stage_path_range_ring_wraps(stager, tmpd):
    """a file of more than 32 pieces: the ring's slots are reused while earlier pieces' copies are in flight"""
    P = S.RING_PIECE
    path = os.path.join(tmpd, "wrap.bin")
    n = (S.RING_SLOTS + 1) * P + 4321
    write_positional(path, n)
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    try:
        for begin, end in ((0, -1), (P + 1, -1), (15, 15 + S.RING_SLOTS * P + 1)):
            check_staged(stager, path, mm, begin, end)
    finally:
        del mm
        os.unlink(path)


# ---- 2. the one-rank C-ABI ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fastq_long_crlf_1", "fastq_tiny_shards_crlf_False", "fasta_crlf",
                                  "fasta_with_lead_False", "fasta_full_name", "fasta_general"])
def test_scan_sharded_one_rank_equals_scan(name):
    """fxg_scan_sharded without a communicator: the same rows (byte for byte), stats and shard info as
    fxg_fasta_scan / fxg_fastq_scan, with and without full_name"""
    lay = S.layout(name)
    eng = engine.get_engine(0)
    f = eng.stage_bytes(lay.data)
    try:
        for full_name in (False, True):
            rows, st, infos = eng.scan_sharded(None, f, lay.mode, full_name=full_name)
            if lay.mode == 0:
                want_rows, want_st = eng.fasta_scan(f, full_name=full_name)
            else:
                want_rows, want_st = eng.fastq_scan(f)
            assert rows.tobytes() == want_rows.tobytes(), (name, full_name)
            assert st == want_st, (name, full_name)
            assert len(infos) == 1
            want = S.shard_info(lay.data, 0, lay.mode)
            for k, v in want.items():
                assert np.asarray(infos[0][k]).tolist() == v, (name, full_name, k)
            exp_rows = fxo.fasta_scan(lay.data, full_name)[0] if lay.mode == 0 else fxo.fastq_scan(lay.data)[0]
            assert_rows_equal(rows, exp_rows, name)
    finally:
        f.free()


def test_shard_exchange_without_comm_copies():
    """fxg_shard_exchange(ctx, NULL, ...) copies the send buffer to the receive buffer"""
    eng = engine.get_engine(0)
    rng = np.random.default_rng(3)
    for nbytes in (128, 100, 1 << 20):
        src = rng.integers(0, 256, size=nbytes, dtype=np.uint8)
        send = eng.upload_rows(src)
        recv = eng.dev_alloc(nbytes)
        try:
            _cabi.check(_cabi.lib().fxg_shard_exchange(eng.ctx, None, C.c_void_p(send.devptr), C.c_void_p(recv.devptr),
                                                       nbytes))
            eng.sync()
            out = np.zeros(nbytes, np.uint8)
            _cabi.check(_cabi.lib().fxg_rows_download(eng.ctx, recv.devptr, nbytes, 1, out.ctypes.data))
            assert np.array_equal(out, src), nbytes
        finally:
            send.free()
            recv.free()


# ---- 3. the loop-back emulation of N ranks ---------------------------------------------------------------
def check_emulation(lay, pts, res, infos, C, what):
    data, mode = lay.data, lay.mode
    exp_rows, exp_total, exp_lines, exp_names = expected(lay.id)
    world = len(pts) - 1
    rows = np.concatenate([p["rows"] for p in res])
    got = rows.copy()
    for f in OFFSET_FIELDS[mode]:
        got[f] -= C                                      # offsets shift by C, nothing else changes
    assert_rows_equal(got, exp_rows, what)
    assert sum(p["stats"]["total_len"] for p in res) == exp_total, what
    if mode == 1:
        assert int(infos["n_lines"].sum()) == exp_lines, what
        _, _, owned, _ = shard.fastq_layout(infos["n_lines"])
    lines_before = 0
    for r in range(world):
        a, b = pts[r], pts[r + 1]
        s = data[a:b]
        want = S.shard_info(s, a + C, mode)
        for k, v in want.items():
            assert np.asarray(infos[r][k]).tolist() == v, (what, r, k, infos[r][k], v)
        assert res[r]["infos"].tobytes() == infos.tobytes(), (what, r)
        st = res[r]["stats"]
        if mode == 0:
            assert len(res[r]["rows"]) == want["n_rows"], (what, r)
            assert (st["lead_lines"], st["lead_bytes"]) == S.fasta_lead(s), (what, r)
        else:
            assert len(res[r]["rows"]) == owned[r], (what, r)
            assert st["lead_lines"] == lines_before, (what, r)
        lines_before += want["n_lines"]
    names = sum((S.split_names(p["names"], p["name_off"]) for p in res), [])
    assert names == exp_names, what
    return rows


def check_fetch(eng, stager, lay, path, res):
    """reads (FASTQ) / extraction (FASTA) on the merged rows: a sample in every shard and every read or record
    next to a cut, against the oracle on the whole file"""
    rows = np.concatenate([p["rows"] for p in res])
    if not len(rows):
        return
    exp_rows = expected(lay.id)[0]
    rng = np.random.default_rng(len(rows))
    ids, first = [], 0
    for p in res:
        k = len(p["rows"])
        if k:
            ids += [first, first + k - 1, first + int(rng.integers(0, k))]
        if first + k < len(rows):
            ids.append(first + k)
        first += k
    ids = np.array(sorted(set(ids)), dtype=np.int64)
    dfile = stager.stage_path(path)
    drows = eng.upload_rows(rows)
    try:
        if lay.mode == 1:
            seq, qual, off = eng.reads(dfile, drows, ids, rlens=rows["rlen"][ids])
            for i, rid in enumerate(ids):
                es, eq = fxo.read_fetch(lay.data, exp_rows[rid])
                assert seq[off[i]:off[i + 1]].tobytes() == es, (lay.name, int(rid))
                assert qual[off[i]:off[i + 1]].tobytes() == eq, (lay.name, int(rid))
        else:
            slen = exp_rows["slen"][ids]
            s = np.concatenate([np.zeros_like(slen), slen // 3])
            e = np.concatenate([slen, np.minimum(slen, slen // 3 + 1000)])
            rid = np.concatenate([ids, ids])
            fl = np.tile(np.array([0, _cabi.X_REVERSE | _cabi.X_COMPLEMENT], np.int32), len(rid))[:len(rid)]
            out, off, _ = eng.extract(dfile, drows, rid, s, e, fl)
            eo, eoff, _ = fxo.subseq_batch(lay.data, exp_rows, rid, s, e, fl)
            assert np.array_equal(off, eoff) and np.array_equal(out, eo), lay.name
    finally:
        drows.free()
        dfile.free()


@pytest.mark.parametrize("name", S.layout_ids())
def test_loopback_layouts(name, engs, stager, tmpd):
    """each layout's own cuts (base offsets as found, then shifted by 2^33), then the split points of worlds
    2, 3, 5, 8, 16; every rank's buffer staged from the file by byte range"""
    lay = S.layout(name)
    path = lay.write(tmpd)
    eng = engine.get_engine(0)
    res, infos = S.emulate(engs, lay.pts, lay.mode, path=path, stager=stager, full_name=lay.full_name)
    base_rows = check_emulation(lay, lay.pts, res, infos, 0, (name, "cuts"))
    check_fetch(eng, stager, lay, path, res)
    res, infos = S.emulate(engs, lay.pts, lay.mode, path=path, stager=stager, full_name=lay.full_name, C=BIG_BASE)
    rows = check_emulation(lay, lay.pts, res, infos, BIG_BASE, (name, "cuts + 2^33"))
    for f in rows.dtype.names:
        assert np.array_equal(rows[f] - (BIG_BASE if f in OFFSET_FIELDS[lay.mode] else 0), base_rows[f]), f
    for world in WORLDS:
        pts = shard.split_points_path(path, world, lay.mode == 0)
        res, infos = S.emulate(engs, pts, lay.mode, path=path, stager=stager, full_name=lay.full_name)
        check_emulation(lay, pts, res, infos, 0, (name, world))


# ---- 4. split_point_dev ------------------------------------------------------------------------------------
def test_split_point_dev_step_edges():
    """the answer on the edges (+-1) of the kernel's 4096-byte steps, counted from from - 1, and from many steps
    before the answer (inside a long line, and past newlines that do not start a header)"""
    rng = np.random.default_rng(91)
    long_line = b">h0\n" + S._seq(rng, 50000) + b"\n"
    wrapped = b">h0\n" + b"".join(S._seq(rng, 4095) + b"\n" for _ in range(12))
    eng = engine.get_engine(0)
    for head in (long_line, wrapped):
        data = head + b">h1 x\nACGT\nAC\n>h2\nA\n"
        x = len(head) - 1                                # '\n' followed by '>'
        f = eng.stage_bytes(data)
        try:
            froms = set(range(x - 40, x + 4)) | set(range(0, 40)) | {len(data) - 1, len(data), len(data) + 3}
            for k in range(0, 8):
                for d in (-2, -1, 0, 1, 2):
                    froms.add(x + 1 - k * S.SPLIT_STEP + d)
            froms |= set(range(1, x, 997))
            for start in sorted(v for v in froms if v >= 0):
                for hdr in (True, False):
                    assert eng.split_point(f, start, hdr) == shard.split_point_bytes(data, start, hdr), (start, hdr)
        finally:
            f.free()


# ---- 5. build_index_sharded and the .fxi -------------------------------------------------------------------
def load_index(path, mode):
    con, rows, pn, stat = (fxi.load_fasta_index if mode == 0 else fxi.load_fastq_index)(path)
    con.close()
    return rows, pn, stat


def assert_same_index(got_path, want_path, mode, what):
    g_rows, g_pn, g_stat = load_index(got_path, mode)
    w_rows, w_pn, w_stat = load_index(want_path, mode)
    assert_rows_equal(g_rows, w_rows, what)
    assert np.array_equal(g_pn.off, w_pn.off) and g_pn.blob.tobytes() == w_pn.blob.tobytes(), what
    assert tuple(g_stat) == tuple(w_stat), what


INDEX_LAYOUTS = ["fasta_crlf", "fasta_full_name", "fastq_long_crlf_3", "fastq_tiny_shards_lf_True",
                 "fastq_read_over_block", "blocks_layout_fasta"]


@pytest.mark.parametrize("name", INDEX_LAYOUTS)
def test_build_index_sharded_writes_the_same_fxi(name, engs, stager, tmpd):
    """one process (a world of one) through shard.build_index_sharded, and a world of 5 merged by hand, write the
    .fxi that Fasta / Fastq write: rows, names, stat (for FASTQ: read count from the line count)"""
    from pyfastx_b200 import api
    lay = S.layout(name)
    path = lay.write(tmpd)
    want = os.path.join(tmpd, name + ".want.fxi")
    if not os.path.exists(want):
        obj = api.Fasta(path, index_file=want, full_name=lay.full_name) if lay.mode == 0 else api.Fastq(path, index_file=want)
        del obj
    got = os.path.join(tmpd, name + ".one.fxi")
    if os.path.exists(got):
        os.unlink(got)
    res = shard.build_index_sharded(path, lay.fmt, index_file=got, full_name=lay.full_name)
    assert res["range"] == (0, len(lay.data))
    assert_same_index(got, want, lay.mode, (name, 1))
    pts = shard.split_points_path(path, 5, lay.mode == 0)
    res, infos = S.emulate(engs, pts, lay.mode, path=path, stager=stager, full_name=lay.full_name)
    check_emulation(lay, pts, res, infos, 0, (name, 5))
    rows, blob, noff = S.merged_index(res)
    total = sum(int(p["stats"]["total_len"]) for p in res)
    merged = os.path.join(tmpd, name + ".five.fxi")
    if os.path.exists(merged):
        os.unlink(merged)
    if lay.mode == 0:
        fxi.write_fasta_index_packed(merged, rows, blob, noff, total).close()
    else:
        fxi.write_fastq_index_packed(merged, rows, blob, noff, int(infos["n_lines"].sum()), total).close()
    assert_same_index(merged, want, lay.mode, (name, 5))
