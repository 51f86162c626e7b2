"""CPU companion of test_full_stats_gpu.py: the statslib restatements give the reference's answers
(tests/golden/full_stats.json.gz, written by tests/golden/make_golden_full_stats.py) and agree with the plain edgelib
versions, the statslib inputs reach the kernel edges they are built for, and the constants they assume are the ones in
csrc/fxg_stats.cu."""
import functools
import gzip
import json
import os
import re

import numpy as np
import pytest

import edgelib as E
import gen
import goldenlib as G
import statslib as S
from oracle import fxo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

with gzip.open(os.path.join(G.GOLD, "full_stats.json.gz"), "rt") as _f:
    GOLD = json.load(_f)


@functools.lru_cache(maxsize=1)
def many_records():
    data = S.many_records()
    return data, fxo.fasta_scan(data)[0]


def fastq_input(name):
    """the bytes of a FASTQ input of the golden file by its name"""
    if name == "many_reads":
        return S.many_reads()
    if name.startswith("inner_cr/"):
        return S.INNER_CR[name.split("/")[1]]
    kind, tag, which = name.split("/")
    eol = b"\r\n" if tag == "crlf" else b"\n"
    return S.quality_classes(eol)[which] if kind == "quality_classes" else S.step_sweep(eol, which)


# ---------------------------------------------------------------------------------------------
# constants
# ---------------------------------------------------------------------------------------------
def test_constants_match_the_source():
    with open(os.path.join(ROOT, "pyfastx_b200", "csrc", "fxg_stats.cu")) as fh:
        src = fh.read()
    assert re.search(r"constexpr int CT_SUB = (\d+);", src).group(1) == str(S.CT_SUB)
    assert re.search(r"constexpr int CT_WARPS = (\d+);", src).group(1) == str(S.CT_WARPS)
    assert re.search(r"const int64_t BATCH = \(int64_t\)1 << (\d+);", src).group(1) == str(S.BATCH.bit_length() - 1)
    # fq_line: 16 bytes per lane from the line start rounded down to 16, then 512-byte steps
    assert "for (int64_t o0 = s & ~(int64_t)15; !done; o0 += %d)" % S.STEP in src
    assert "const int64_t o = o0 + lane * %d;" % S.LANE in src
    assert "done = has != 0 || o0 + %d >= n;" % S.STEP in src
    # the stats launch: sm_count * 8 CTAs of 256 threads, a warp per read
    launch = re.search(r"fastq_stats_kernel<<<ctx->sm_count \* (\d+), (\d+), ", src)
    assert launch.groups() == (str(S.STATS_CTAS_PER_SM), str(S.STATS_THREADS))
    assert "__launch_bounds__(%d) fastq_stats_kernel" % S.STATS_THREADS in src
    assert S.stats_warps() == 8448
    # a composition batch counts 3 launches of its own and the 3 of the offset prefix (test_full_stats_gpu.py)
    assert src.count("ctx->launches += 3;") == 1 and "fxg_extract_plan_dev(ctx, d_zero, d_cnt, nb, d_off" in src
    with open(os.path.join(ROOT, "pyfastx_b200", "csrc", "fxg_extract.cu")) as fh:
        assert "FxgProfScope prof(ctx, FXG_PROF_PLAN, 3);" in fh.read()


# ---------------------------------------------------------------------------------------------
# the restatements give the reference's answers
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(GOLD["fastq"]))
def test_fastq_restatement_gives_the_references_answers(name):
    exp = GOLD["fastq"][name]
    got = S.fastq_answers(fastq_input(name))
    assert {k: got[k] for k in exp} == exp


def test_fasta_restatement_gives_the_references_answers():
    for name, exp in sorted(GOLD["fasta"].items()):
        if name == "many_records":
            data, rows = many_records()
        else:
            data = S.tile_sweep(big=0, ascii_only=True)
            rows = fxo.fasta_scan(data)[0]
        comp, total = S.composition(data, rows)
        assert S.comp_digest(S.comp_table(comp, total)) == exp["comp_digest"], name
        assert S.fasta_getters(total) == {k: exp[k] for k in ("composition", "gc_content", "gc_skew", "type")}, name


# ---------------------------------------------------------------------------------------------
# ... and the plain edgelib restatements on seeded inputs
# ---------------------------------------------------------------------------------------------
def _fastq_small():
    yield "random", gen.random_fastq(1, n_reads=300)
    yield "random_crlf_tail", gen.random_fastq(2, n_reads=300, crlf=True, partial_tail=2)
    yield "random_nonl", gen.random_fastq(3, n_reads=300, partial_tail=1, no_trailing_newline=True)
    for eol in (b"\n", b"\r\n"):
        for name, data in sorted(S.quality_classes(eol).items()):
            yield name, data
        for end in S.STEP_ENDS:
            yield "step_" + end, S.step_sweep(eol, end)
    # '\r' inside a quality line and doubled: the reference's walk stops early
    yield "inner_cr", b"@a\nACGT\n+\nI\r!~\n@b\nAC\n+\n#\r\r\n@c\nA\r\n+\n\r\r\r\n@d\nA\n+\n\x7f\rJ\r\n"
    for name, data in sorted(S.INNER_CR.items()):
        yield "inner_cr_" + name, data


@pytest.mark.parametrize("case", list(_fastq_small()), ids=lambda c: c[0])
def test_fastq_stats_matches_edgelib(case):
    name, data = case
    got = S.fastq_stats(data)
    got.pop("phred")
    assert got == E.fastq_stats(data)


def test_composition_matches_edgelib():
    for data in (S.many_records(20000, long_at=(5000, 5001)), S.tile_sweep(big=0), gen.random_fasta(4, n_records=300)):
        rows = fxo.fasta_scan(data)[0]
        comp, total = S.composition(data, rows, chunk_rows=997, chunk_bytes=50000)
        exp, exp_total = E.composition(data, rows)
        assert comp.tolist() == exp and np.array_equal(total, exp_total)


def test_encoding_type_and_phred_restated():
    assert S.encoding_type(35, 70) == ["Sanger Phred+33", "Illumina 1.8+ Phred+33", "PacBio HiFi Phred+33"]
    assert S.encoding_type(66, 104) == ["Solexa Solexa+64", "Illumina 1.3+ Phred+64", "Illumina 1.5+ Phred+64",
                                       "PacBio HiFi Phred+33"]
    assert S.encoding_type(32, 70) == S.encoding_type(40, 127) == ["Unknown"]
    assert [S.phred({"minqs": lo, "maxqs": hi}) for lo, hi in ((58, 100), (59, 100), (59, 74), (59, 75))] == [33, 64, 0, 64]


# ---------------------------------------------------------------------------------------------
# the inputs reach their targets
# ---------------------------------------------------------------------------------------------
def test_many_records_crosses_the_batch_edges():
    data, rows = many_records()
    assert len(rows) == S.MANY_RECORDS > 2 * S.BATCH
    end = rows["boff"] + rows["blen"]
    for r in S.LONG_AT:
        assert rows["slen"][r] == S.LONG_LEN and rows["blen"][r] > 3 * S.CT_SUB
    for b in (S.BATCH, 2 * S.BATCH):
        # one sub-tile holds the last bytes of record b - 1 (one batch) and the first of record b (the next)
        assert (end[b - 1] - 1) // S.CT_SUB == rows["boff"][b] // S.CT_SUB
        assert (end[b - 1] - 1) % S.CT_SUB != S.CT_SUB - 1
    assert (rows["elen"] == 2).sum() > len(rows) // 10 and (rows["slen"] == 0).sum() > len(rows) // 20
    comp, total = S.composition(data[:rows["boff"][20000]], rows[:20000])
    assert np.count_nonzero(total) > 30                              # mixed alphabets


def test_tile_sweep_reaches_every_offset():
    data = S.tile_sweep()
    rows = fxo.fasta_scan(data)[0]
    starts = {int(b): int(n) for b, n in zip(rows["boff"], rows["blen"])}
    ends = set((rows["boff"] + rows["blen"])[rows["blen"] > 0].tolist())
    for k, d, kind in S.sweep_sites():
        at = k * S.CT_SUB + d
        if kind == "end":
            assert at in ends, (k, d)
        elif kind == "start":
            assert starts.get(at, 0) > 0, (k, d)
        else:
            assert starts.get(at) == 0, (k, d)
    sites = S.sweep_sites()
    assert {(d, kind, k % 2) for k, d, kind in sites} == {(d, kind, p) for d in S.SWEEP for kind in ("end", "start", "empty")
                                                         for p in (0, 1)}
    assert {d % 16 for d in S.SWEEP} == set(range(16))
    assert rows["blen"].max() >= 64 << 20
    lines = np.frombuffer(data, np.uint8)[int(rows["boff"][1]):]
    assert set(np.unique(lines).tolist()) == set(range(256))
    assert len(rows) == data.count(b"\n>") + 1                      # '>' starts no sequence line


def test_quality_classes_cover_every_threshold():
    got = {}
    for eol in (b"\n", b"\r\n"):
        for name, data in S.quality_classes(eol).items():
            got[name, eol] = S.fastq_stats(data)
    qs = [(st["minqs"], st["maxqs"]) for st in got.values()]
    for v in (32, 33, 58, 59, 63, 64, 65, 66):
        assert any(lo == v for lo, _ in qs), v
    for v in (73, 74, 75, 104, 105, 126, 127):
        assert any(hi == v for _, hi in qs), v
    assert {st["phred"] for st in got.values()} == {0, 33, 64}
    possible = {tuple(S.encoding_type(lo, hi)) for lo in range(-128, 128) for hi in range(lo, 128)}
    assert {tuple(S.encoding_type(lo, hi)) for lo, hi in qs} == possible
    assert min(lo for lo, _ in qs) == -128 and got["high_byte_ff", b"\n"]["minqs"] == -1
    assert got["above_104", b"\n"]["minqs"] == 104 and got["below_33", b"\n"]["maxqs"] == 33


@pytest.mark.parametrize("eol", [b"\n", b"\r\n"], ids=["lf", "crlf"])
def test_step_sweep_reaches_every_length_and_alignment(eol):
    e = len(eol)
    for end in S.STEP_ENDS:
        data = S.step_sweep(eol, end)
        a = np.frombuffer(data, np.uint8)
        starts, ends = S.lines(data)
        k = np.arange(starts.size)
        sq, ql = starts[k % 4 == 1], starts[k % 4 == 3]
        slen = ends[k % 4 == 1] - sq - (e - 1)
        assert set(slen.tolist()) >= set(S.STEP_LENGTHS)
        assert {int(s) % 16 for s in sq} == set(range(16)) and {int(s) % 16 for s in ql} == set(range(16))
        assert {int(n) % S.STEP for n in slen} == set(range(S.STEP))
        if e == 2:
            # '\r' as the last byte of a lane and as the last byte of a step of the line's walk
            full = np.concatenate([sq, ql])
            fend = np.concatenate([ends[k % 4 == 1], ends[k % 4 == 3]]) - 1
            full, fend = full[fend < a.size - 1], fend[fend < a.size - 1]           # lines that end in CRLF
            assert (a[fend] == 13).all()
            assert (fend % 16 == 15).any() and ((fend - (full & ~15)) % S.STEP == S.STEP - 1).any()
        if end in ("nl", "nonl"):
            assert starts.size % 4 == 0 and (data[-1:] == b"\n") == (end == "nl")
            assert (a.size - (int(ql[-1]) & ~15)) % S.STEP == 0
        else:
            assert starts.size % 4 == int(end[-1])


def test_many_reads_puts_the_extremes_before_the_last_round():
    data = S.many_reads()
    st = S.fastq_stats(data)
    rows, _, _ = fxo.fastq_scan(data)
    n = len(rows)
    assert n == S.MANY_READS >= 40 * S.stats_warps()
    m = S.many_reads_marks()
    a = np.frombuffer(data, np.uint8)
    qmin = np.array([a[q:q + r].min() for q, r in zip(rows["qoff"][m["minq"] - 50:m["maxq"] + 50],
                                                     rows["rlen"][m["minq"] - 50:m["maxq"] + 50])])
    assert (st["minqs"], st["maxqs"], st["minlen"], st["maxlen"]) == (34, 72, 3, 400)
    assert (rows["rlen"] == 3).sum() == 1 and rows["rlen"][m["short"]] == 3
    assert (rows["rlen"] == 400).sum() == 1 and rows["rlen"][m["long"]] == 400
    assert (qmin == 34).sum() == 1 and qmin[50] == 34
    assert data.count(b"\x22") == 1 and data.count(b"\x48") == 1              # quality 34 ('"') and 72 ('H') once each
    for i in m.values():
        # each is in the round before the last of 8,448 warps, and has a later read in its warp up to 12,000 warps
        assert n - 2 * S.stats_warps() <= i < n - S.stats_warps() and i + 12000 < n
