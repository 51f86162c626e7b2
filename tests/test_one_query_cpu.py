"""CPU companion of test_one_query_gpu.py: its thresholds are the ones in csrc/fxg_extract.cu, and every layout,
query set and schedule it runs is what it claims to be, checked against the oracle alone."""
import os
import re

import numpy as np

import onequerylib as Q
from oracle import fxo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pyfastx_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as fh:
        return fh.read()


def test_thresholds_match_the_source():
    src = _src("fxg_extract.cu")
    # the service limit, in both one-query entry points
    assert re.findall(r"direct && svc_enabled\(\) && (?:len|rlen) <= (\d+)\)", src) == [str(Q.SVC_LIMIT)] * 2
    # output straight to mapped pinned memory up to ONE_PINNED, in both
    assert re.findall(r"const int64_t ONE_PINNED = 1 << (\d+);", src) == [str(Q.ONE_PINNED.bit_length() - 1)] * 2
    # the 2048-byte piece: the service kernel and extract_one_kernel's host side
    assert re.findall(r"warps = \(len \+ (\d+)\) / (\d+);", src) == [(str(Q.PIECE - 1), str(Q.PIECE))] * 2
    xthreads = int(re.search(r"constexpr int XTHREADS = (\d+);", src).group(1))
    assert re.search(r"constexpr int XWARPS = XTHREADS / 32;", src) and xthreads // 32 == Q.XWARPS
    # the piece cap of the launch path, and the service's cap at its own warps
    assert re.search(r"const int64_t maxw = \(int64_t\)ctx->sm_count \* (\d+) \* XWARPS;", src).group(1) == str(Q.CTAS_PER_SM)
    assert "if (warps > XWARPS) warps = XWARPS;" in src
    assert Q.threshold(132) == 8_650_752
    # the file pool keeps freed buffers of at least 64 MiB (the interleaving test hands one over)
    assert "cap >= ((int64_t)64 << 20)" in _src("fxg_api.cu")
    assert re.search(r"PINNED_CHUNK = \(size_t\)(\d+) << 20;", _src("fxg_api.cu")).group(1) == str(Q.PINNED_CHUNK >> 20)


def record_lines(data, row):
    """lengths of the sequence lines of one record (end of line included), from the bytes"""
    a = np.frombuffer(data, np.uint8)
    b0 = int(row["boff"])
    b1 = min(b0 + int(row["blen"]), a.size)
    nl = np.flatnonzero(a[b0:b1] == 10) + 1
    ends = np.concatenate([nl, [b1 - b0]]) if (nl.size == 0 or nl[-1] != b1 - b0) else nl
    return np.diff(np.concatenate([[0], ends]))


def test_fasta_layouts_against_the_oracle():
    data, layouts = Q.fasta_layouts(Q.NOMINAL_SMS)
    rows, total, _ = fxo.fasta_scan(data)
    assert len(rows) == len(layouts) and total == sum(x["slen"] for x in layouts)
    assert len(data) >= 64 << 20                                       # pooled on free
    assert not data.endswith(b"\n")                                     # the last record has no trailing newline
    for r, lay in zip(rows, layouts):
        assert int(r["slen"]) == lay["slen"] and int(r["norm"]) == lay["norm"], lay["name"]
        ln = record_lines(data, r)
        uniform = bool((ln[:-1] == ln[0]).all() and ln[-1] <= ln[0])   # the scan's pad[0] & 1
        assert uniform == bool(lay["uniform"]), lay["name"]
        seq = fxo.subseq(data, r, 0, lay["slen"])
        a = np.frombuffer(seq, np.uint8)
        assert (a >= 97).any() and (a < 97).any() and np.isin(a & 0xDF, Q.IUPAC).any(), lay["name"]
        assert max(lay["lengths"]) == lay["slen"]
    by = {x["name"]: (r, x) for r, x in zip(rows, layouts)}
    assert by["crlf80"][0]["elen"] == 2 and by["crlf80"][0]["llen"] == 82
    assert record_lines(data, by["longlast"][0])[-1] > 60 + 1 and by["blank"][0]["norm"] == 0
    assert by["oneline"][0]["llen"] == by["oneline"][1]["slen"] + 1
    # every length the issue of the paths turns on, at every start, on a record long enough for it
    t = Q.threshold(Q.NOMINAL_SMS)
    want = {1, 15, 16, 17, 2047, 2048, 2049, 16383, 16384, 16385, 65535, 65536, 65537, (1 << 20) - 1, 1 << 20,
            (1 << 20) + 1, t - 16, t, t + 1, t + 16, Q.BIG_SLICE}
    assert want <= set(by["lf60"][1]["lengths"]) and want - {Q.BIG_SLICE} <= set(by["crlf80"][1]["lengths"])
    q = Q.fasta_queries(layouts, rows)
    paths = {Q.path_of(e - s) for _, s, e, _ in q}
    assert paths == {"service", "mapped", "device"}
    for i, s, e, f in q:
        assert 0 <= s < e <= int(rows["slen"][i])
    starts = {(i, e - s): set() for i, s, e, _ in q}
    for i, s, e, _ in q:
        starts[(i, e - s)].add(s)
    for (i, n), ss in starts.items():
        slen = int(rows["slen"][i])
        assert {0, slen - n} <= ss and (n == slen or any(x % 2 == 1 for x in ss)), (i, n)
    # a slice in the longer last line is not what the covering-range formula of a split piece would give: a split
    # would show (the launch path must not split this record)
    r, _ = by["longlast"]
    n = 65537
    s = int(r["slen"]) - n
    whole = fxo.subseq(data, r, s, s + n)
    pieces = b"".join(fxo.subseq(data, r, a, min(a + Q.PIECE, s + n)) for a in range(s, s + n, Q.PIECE))
    assert whole != pieces


def test_fastq_files_against_the_oracle():
    for eol, trailing in ((b"\n", False), (b"\r\n", True)):
        data = Q.fastq_file(Q.FASTQ_LENGTHS, eol=eol, trailing=trailing)
        rows, size, nlines = fxo.fastq_scan(data)
        assert [int(x) for x in rows["rlen"]] == Q.FASTQ_LENGTHS and nlines == 4 * len(Q.FASTQ_LENGTHS)
        assert data.endswith(eol) == trailing
        assert {Q.path_of(n) for n in Q.FASTQ_LENGTHS} == {"service", "mapped", "device"}
        qual = b"".join(fxo.read_fetch(data, r)[1] for r in rows)
        assert set(qual) == set(range(33, 127))
        for r in rows[:3]:
            sq, ql = fxo.read_fetch(data, r)
            assert Q.read_expected(data, r, 1, Q.UPPER | Q.RC) == ql[::-1]
            assert Q.read_expected(data, r, 0, Q.RC) == bytes(fxo.complement_lut()[np.frombuffer(sq, np.uint8)][::-1])


def test_schedule_against_the_oracle():
    data, layouts = Q.fasta_layouts(Q.NOMINAL_SMS)
    rows = fxo.fasta_scan(data)[0]
    fqd = Q.fastq_file(Q.FASTQ_LENGTHS, trailing=False)
    qrows = fxo.fastq_scan(fqd)[0]
    sets = {"A": (rows["slen"], False), "Aup": (rows["slen"], True), "B": (rows["slen"], False)}
    sched = Q.schedule(2000, sets, qrows["rlen"])
    assert sched == Q.schedule(2000, sets, qrows["rlen"])              # seeded

    def path(it):
        return Q.path_of(it[4] - it[3] if it[0] == "fa" else int(qrows["rlen"][it[1]]))

    kinds = [it[0] for it in sched]
    assert kinds.count("fq") > 400 and {it[1] for it in sched if it[0] == "fa"} == set(sets)
    assert all(path(a) != path(b) or a[0] != b[0] for a, b in zip(sched, sched[1:]))
    for kind in ("fa", "fq"):
        assert {path(it) for it in sched if it[0] == kind} == {"service", "mapped", "device"}
    for it in sched[::7]:
        if it[0] == "fa":
            _, key, i, s, e, f = it
            assert 0 <= s < e <= int(rows["slen"][i]) and f in Q.GETTERS
            assert len(fxo.subseq(data, rows[i], s, e, f | (Q.UPPER if sets[key][1] else 0))) == e - s
        else:
            _, i, which, f = it
            assert len(Q.read_expected(fqd, qrows[i], which, f)) == int(qrows["rlen"][i]) and (f == 0 or not which)


def test_upload_order_data_against_the_oracle():
    data, frows, qrows = Q.upload_order_data()
    assert len(data) > Q.PINNED_CHUNK + (16 << 20)                      # the last pinned chunk holds the queried bytes
    s, e = Q.UPLOAD_QUERY
    assert e - s <= Q.SVC_LIMIT and int(frows["slen"][-1]) == 70_001 and e <= 70_001
    assert int(frows["boff"][-1]) > Q.PINNED_CHUNK and int(qrows["soff"][-1]) > Q.PINNED_CHUNK
    sq, ql = fxo.read_fetch(data, qrows[-1])
    assert len(sq) == len(ql) == 60_000 and int(qrows["rlen"][-1]) <= Q.SVC_LIMIT
    assert fxo.subseq(data, frows[-1], s, e) != b"N" * (e - s)
