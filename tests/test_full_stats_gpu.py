"""Full-index statistics (K7, csrc/fxg_stats.cu) past the inputs of test_stats_gpu.py: more than two composition
batches, record edges at every offset around the 8 KiB sub-tiles, a 64 MiB record, base_offset slices, every quality
class, lines across fq_line's 512-byte steps, and more reads than the launch has warps.

The kernels get the CPU oracle's rows (oracle/fxo), so a failure points at K7 and not at the scan; answers are
compared with the statslib restatements and, where the reference could run, with tests/golden/full_stats.json.gz."""
import functools
import gzip
import json
import os
import sqlite3

import numpy as np
import pytest

import goldenlib as G
import statslib as S
import pyfastx_b200 as pyfastx
from oracle import fxo
from pyfastx_b200 import _cabi, engine

pytestmark = pytest.mark.gpu

with gzip.open(os.path.join(G.GOLD, "full_stats.json.gz"), "rt") as _f:
    GOLD = json.load(_f)

META = ("a", "c", "g", "t", "n", "maxlen", "minlen", "minqs", "maxqs", "phred")


def launches(eng):
    return _cabi.lib().fxg_ctx_launch_count(eng.ctx)


def triplets(comp):
    """COMP_ROW array -> int64[n, 3] for np.array_equal"""
    return np.stack([comp["seqid"], comp["abc"], comp["num"]], axis=1).astype(np.int64)


def fxi_comp(path):
    """the `comp` table of an index file, in ID order -> int64[n, 3]"""
    con = sqlite3.connect(path)
    cur = con.execute("SELECT seqid,abc,num FROM comp ORDER BY ID")
    parts = []
    while True:
        chunk = cur.fetchmany(1 << 20)
        if not chunk:
            break
        parts.append(np.array(chunk, np.int64))
    con.close()
    return np.concatenate(parts) if parts else np.zeros((0, 3), np.int64)


@functools.lru_cache(maxsize=1)
def many_records():
    data = S.many_records()
    rows = fxo.fasta_scan(data)[0]
    comp, total = S.composition(data, rows)
    return data, rows, comp, total


@functools.lru_cache(maxsize=1)
def tile_sweep():
    data = S.tile_sweep()
    rows = fxo.fasta_scan(data)[0]
    return data, rows


def composition_on_gpu(eng, data, rows, base_offset=0):
    f = eng.stage_bytes(data)
    dr = eng.upload_rows(rows)
    try:
        return eng.fasta_composition(f, dr, base_offset=base_offset)
    finally:
        dr.free()
        f.free()


def fastq_rows(data):
    """the oracle's rows of the complete reads, plus the row of a trailing partial record's sequence line (the
    reference counts its bases) -> (rows, n_complete, trailing)"""
    rows, _, n_lines = fxo.fastq_scan(data)
    n = len(rows)
    trailing = n_lines % 4 >= 2
    if trailing:
        tail = np.zeros(1, _cabi.FASTQ_ROW)
        tail["soff"] = S.lines(data)[0][4 * n + 1]
        rows = np.concatenate([rows, tail])
    return rows, n, trailing


def fastq_stats_on_gpu(eng, data, base_offset=0, rows=None):
    if rows is None:
        rows, n, trailing = fastq_rows(data)
    else:
        n, trailing = len(rows), False
    f = eng.stage_bytes(data)
    dr = eng.upload_rows(rows)
    try:
        return eng.fastq_stats(f, dr, n, base_offset=base_offset, trailing_seq=trailing)
    finally:
        dr.free()
        f.free()


# ---------------------------------------------------------------------------------------------
# FASTA composition
# ---------------------------------------------------------------------------------------------
def test_many_records_three_batches(tmp_path):
    eng = engine.get_engine(0)
    data, rows, comp, total = many_records()
    f = eng.stage_bytes(data)
    dr = eng.upload_rows(rows)
    n0 = launches(eng)
    got, got_total = eng.fasta_composition(f, dr)
    # each batch counts 6 launches: hist + count + emit, and the three kernels of fxg_extract_plan_dev's offset prefix
    # (test_full_stats_cpu.py::test_constants_match_the_source pins both counters in the source)
    assert launches(eng) - n0 == 6 * 3
    dr.free()
    f.free()
    assert np.array_equal(triplets(got), triplets(comp)) and np.array_equal(got_total, total)
    assert S.comp_digest(S.comp_table(got, got_total)) == GOLD["fasta"]["many_records"]["comp_digest"]

    p = str(tmp_path / "many.fa")
    with open(p, "wb") as fh:
        fh.write(data)
    want = S.fasta_getters(total)
    fa = pyfastx.Fasta(p, full_index=True)
    assert (fa.composition, fa.gc_content, fa.gc_skew, fa.type) == tuple(want[k] for k in ("composition", "gc_content",
                                                                                          "gc_skew", "type"))
    del fa
    table = fxi_comp(p + ".fxi")
    assert np.array_equal(table, triplets(S.comp_table(comp, total)))                 # 128 seqid-0 rows at the end
    del table
    fb = pyfastx.Fasta(p)
    n0 = launches(fb._st.engine)
    assert (fb.composition, fb.gc_content, fb.gc_skew, fb.type) == tuple(want[k] for k in ("composition", "gc_content",
                                                                                          "gc_skew", "type"))
    assert launches(fb._st.engine) == n0                                               # loaded, not recomputed
    gold = GOLD["fasta"]["many_records"]
    assert (fb.composition, fb.gc_content, fb.gc_skew, fb.type) == (gold["composition"], gold["gc_content"],
                                                                    gold["gc_skew"], gold["type"])


def test_tile_sweep_composition():
    data, rows = tile_sweep()
    comp, total = S.composition(data, rows)
    got, got_total = composition_on_gpu(engine.get_engine(0), data, rows)
    assert np.array_equal(triplets(got), triplets(comp)) and np.array_equal(got_total, total)


def test_tile_sweep_ascii_golden():
    data = S.tile_sweep(big=0, ascii_only=True)
    rows = fxo.fasta_scan(data)[0]
    got, got_total = composition_on_gpu(engine.get_engine(0), data, rows)
    exp = GOLD["fasta"]["tile_sweep_ascii"]
    assert S.comp_digest(S.comp_table(got, got_total)) == exp["comp_digest"]
    assert S.fasta_getters(got_total) == {k: exp[k] for k in ("composition", "gc_content", "gc_skew", "type")}


def test_composition_base_offset_slices():
    """three slices of tile_sweep cut at record starts ('>'), each staged on its own with base_offset = its start and
    the rows it wholly holds (global boff): the per-record counts are the whole file's, seqid 1-based per call"""
    eng = engine.get_engine(0)
    data, rows = tile_sweep()
    comp, total = S.composition(data, rows)
    whole = triplets(comp)
    n = len(rows)
    cut_rows = [0, n // 3 + 1, n - 2, n]                       # the last-but-one slice holds the 64 MiB record
    hstart = lambda r: data.rfind(b"\n>", 0, int(rows["boff"][r])) + 1 if r else 0
    cuts = [hstart(r) for r in cut_rows[:-1]] + [len(data)]
    assert rows["blen"][n - 2] >= 64 << 20
    sum_total = np.zeros(128, np.int64)
    for (r0, r1), (lo, hi) in zip(zip(cut_rows, cut_rows[1:]), zip(cuts, cuts[1:])):
        sub = rows[r0:r1]
        assert sub["boff"][0] >= lo and sub["boff"][-1] + sub["blen"][-1] <= hi
        got, got_total = composition_on_gpu(eng, data[lo:hi], sub, base_offset=lo)
        exp = whole[(whole[:, 0] > r0) & (whole[:, 0] <= r1)] - [r0, 0, 0]
        assert np.array_equal(triplets(got), exp), (lo, hi)
        sum_total += got_total
    assert np.array_equal(sum_total, total)


# ---------------------------------------------------------------------------------------------
# FASTQ statistics
# ---------------------------------------------------------------------------------------------
def _check_fastq_file(tmp_path, name, data, gold):
    want = S.fastq_answers(data)
    if gold is not None:
        assert {k: want[k] for k in gold} == gold, name
    m = fastq_stats_on_gpu(engine.get_engine(0), data)
    assert [m[k] for k in META[:5]] == want["base"][0], name
    assert [m[k] for k in META[5:]] == want["meta"][0], name
    p = str(tmp_path / (name.replace("/", "_") + ".fq"))
    with open(p, "wb") as fh:
        fh.write(data)
    fq = pyfastx.Fastq(p, full_index=True)
    got = {"composition": fq.composition, "gc_content": fq.gc_content, "maxlen": fq.maxlen, "minlen": fq.minlen,
           "maxqual": fq.maxqual, "minqual": fq.minqual, "phred": fq.phred, "encoding_type": fq.encoding_type}
    del fq
    con = sqlite3.connect(p + ".fxi")
    got["base"] = [list(r) for r in con.execute("SELECT * FROM base")]
    got["meta"] = [list(r) for r in con.execute("SELECT * FROM meta")]
    con.close()
    assert got == {k: want[k] for k in got}, name
    fb = pyfastx.Fastq(p)                                               # loads base / meta from the .fxi
    assert (fb.composition, fb.maxlen, fb.minlen, fb.maxqual, fb.minqual, fb.phred, fb.encoding_type) == tuple(
        want[k] for k in ("composition", "maxlen", "minlen", "maxqual", "minqual", "phred", "encoding_type")), name


@pytest.mark.parametrize("name", sorted(S.INNER_CR))
def test_inner_cr_in_quality_line(tmp_path, name):
    """a '\r' before a quality line's last byte ends the reference's walk early: the bytes after the stop are not in
    the quality range and the length is the walk's, not the count of bytes other than '\r'"""
    key = "inner_cr/" + name
    _check_fastq_file(tmp_path, key, S.INNER_CR[name], GOLD["fastq"][key])


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_quality_classes(tmp_path, eol):
    tag = "lf" if eol == b"\n" else "crlf"
    for name, data in sorted(S.quality_classes(eol).items()):
        key = "quality_classes/%s/%s" % (tag, name)
        _check_fastq_file(tmp_path, key, data, GOLD["fastq"][key])


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_step_sweep(tmp_path, eol):
    tag = "lf" if eol == b"\n" else "crlf"
    for end in S.STEP_ENDS:
        key = "step_sweep/%s/%s" % (tag, end)
        _check_fastq_file(tmp_path, key, S.step_sweep(eol, end), GOLD["fastq"][key])


def test_many_reads():
    eng = engine.get_engine(0)
    data = S.many_reads()
    nwarps = S.stats_warps(eng.sm_count)
    n = S.MANY_READS
    assert n >= 40 * nwarps and all(i + nwarps < n for i in S.many_reads_marks().values())
    want = S.fastq_answers(data)
    m = fastq_stats_on_gpu(eng, data)
    assert [m[k] for k in META[:5]] == want["base"][0] and [m[k] for k in META[5:]] == want["meta"][0]
    assert want["base"] == GOLD["fastq"]["many_reads"]["base"] and want["meta"] == GOLD["fastq"]["many_reads"]["meta"]


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_fastq_base_offset_slices(eol):
    """a step_sweep file cut at three read starts, each slice staged with base_offset = its start and the rows of the
    reads it holds (global offsets): each gives the statistics of its own bytes"""
    eng = engine.get_engine(0)
    data = S.step_sweep(eol, "nl")
    rows, n, _ = fastq_rows(data)
    starts = S.lines(data)[0]
    cut_reads = [0, n // 3, 2 * n // 3, n]
    cuts = [int(starts[4 * r]) for r in cut_reads[:-1]] + [len(data)]
    for (r0, r1), (lo, hi) in zip(zip(cut_reads, cut_reads[1:]), zip(cuts, cuts[1:])):
        m = fastq_stats_on_gpu(eng, data[lo:hi], base_offset=lo, rows=rows[r0:r1])
        want = S.fastq_stats(data[lo:hi])
        assert {k: m[k] for k in META} == {k: want[k] for k in META}, (lo, hi)


# ---------------------------------------------------------------------------------------------
# compressed inputs: BGZF and plain gzip, the second open through the checkpoints
# ---------------------------------------------------------------------------------------------
def _fasta_full(path):
    fa = pyfastx.Fasta(path, full_index=True)
    out = (fa.composition, fa.gc_content, fa.gc_skew, fa.type)
    del fa
    return out, fxi_comp(path + ".fxi")


def test_compressed_inputs_give_the_plain_statistics(tmp_path):
    eng = engine.get_engine(0)
    data = S.many_records(S.BATCH + 4000, long_at=(S.BATCH - 1, S.BATCH))         # two batches
    rows = fxo.fasta_scan(data)[0]
    comp, total = S.composition(data, rows)
    fq = S.quality_classes(b"\r\n")["high_bytes"]
    fq_want = S.fastq_answers(fq)
    plain = str(tmp_path / "p.fa")
    with open(plain, "wb") as fh:
        fh.write(data)
    want, table = _fasta_full(plain)
    assert np.array_equal(table, triplets(S.comp_table(comp, total)))
    for kind, z in (("bgzf", S.bgzf(data)), ("gzip", S.plain_gzip(data))):
        p = str(tmp_path / ("c.%s.fa.gz" % kind))
        with open(p, "wb") as fh:
            fh.write(z)
        got, got_table = _fasta_full(p)
        assert got == want and np.array_equal(got_table, table), kind
        fb = pyfastx.Fasta(p)                                       # second open: BGZF members / gzip checkpoints
        assert fb.is_gzip and (kind == "bgzf" or fb._st.gzip_path == "gpu-checkpoints")
        assert (fb.composition, fb.gc_content, fb.gc_skew, fb.type) == want
        again, again_total = eng.fasta_composition(fb._st.dfile, fb._drows)
        assert np.array_equal(triplets(again), triplets(comp)) and np.array_equal(again_total, total), kind
        del fb
        q = str(tmp_path / ("c.%s.fq.gz" % kind))
        with open(q, "wb") as fh:
            fh.write(S.bgzf(fq) if kind == "bgzf" else S.plain_gzip(fq))
        f1 = pyfastx.Fastq(q, full_index=True)
        assert (f1.minqual, f1.maxqual, f1.phred, f1.encoding_type, f1.composition) == (
            fq_want["minqual"], fq_want["maxqual"], fq_want["phred"], fq_want["encoding_type"], fq_want["composition"])
        del f1
        f2 = pyfastx.Fastq(q)
        assert f2.is_gzip and (kind == "bgzf" or f2._st.gzip_path == "gpu-checkpoints")
        m = eng.fastq_stats(f2._st.dfile, f2._drows, len(f2._rows))
        assert [m[k] for k in META[:5]] == fq_want["base"][0] and [m[k] for k in META[5:]] == fq_want["meta"][0], kind
        assert (f2.minqual, f2.maxqual, f2.minlen, f2.maxlen) == (fq_want["minqual"], fq_want["maxqual"],
                                                                  fq_want["minlen"], fq_want["maxlen"])
