"""The byte-level edge patterns of tests/edgelib.py placed exactly on the scan's region (2 KiB), FASTQ window (16 KiB)
and prefix-block (8 MiB) edges, at shifts -3..+3, on mark's fast, general and counts-only paths
(test_edge_layouts_cpu.py checks that they get there).  Every input goes through each kernel that reads it, against the
CPU oracle or a plain numpy restatement:

- the scan: every row field, n_rows / total_len (FASTQ: n_lines);
- FASTA extraction of whole records near each anchor and of windows that start at, end at or cross it, under all eight
  upper / reverse / complement flag combinations with A/C/G/T counts, and the one-query service on a sample;
- full-index composition (FASTA) and statistics (FASTQ);
- locate on both strands over every record / read (on the 8 MiB inputs: the FASTA records next to the anchors), and
  locate_approx with one mismatch on the smaller inputs;
- the split-phase scan with cuts next to the first anchor and one byte either side of it: FASTA rows with cuts at the
  header line at or after each point (the anchor itself where the anchor is a header's '>'), the shard infos with cuts
  at the line start at or after each point; FASTQ rows with cuts at the line starts;
- the same bytes as BGZF with a member edge at every anchor."""
import struct
import zlib

import numpy as np
import pytest

import approxlib as AP
import edgelib as E
import searchlib as SL
from oracle import fxo
from pyfastx_b200 import _cabi, engine, shard

from test_fasta_line_record_gpu import shard_info_expected
from test_gpu_parity import assert_rows_equal, emulate_sharded

pytestmark = pytest.mark.gpu

BOTH = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS
PATTERNS = (b"TCAGA", b"GTTGCAAC")         # the last bytes of a 60-column line / the bytes after its first four
APPROX = b"GACCATGG"
FLAGS = tuple(range(8))                   # upper | reverse | complement
SMALL = 1 << 20                           # approximate search only below this size


@pytest.fixture(scope="module")
def eng():
    return engine.get_engine(0)


def bgzf_at(data, edges):
    """BGZF with a member edge at every offset of `edges` (and at least every 0xff00 bytes), plus the EOF member"""
    cuts = sorted({0, len(data), *[e for e in edges if 0 < e < len(data)], *range(0, len(data), 0xff00)})
    out = []
    for a, b in zip(cuts, cuts[1:]):
        chunk = data[a:b]
        co = zlib.compressobj(1, zlib.DEFLATED, -15)
        comp = co.compress(chunk) + co.flush()
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(comp) + 25)
                   + comp + struct.pack("<II", zlib.crc32(chunk), len(chunk)))
    out.append(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))
    return b"".join(out), len(cuts) - 1


def hit_list(hits, approx=False):
    cols = [hits["query"].tolist(), hits["start"].tolist(), hits["minus"].tolist()]
    if approx:
        cols.append(hits["mismatches"].tolist())
    return list(zip(*cols))


def seq_index(data, row, at):
    """sequence coordinate of file offset `at` in a record: bytes of [boff, at) other than '\\n' / '\\r', clipped"""
    boff = int(row["boff"])
    seg = np.frombuffer(data, np.uint8)[boff:max(boff, at)]
    return int(min(max(((seg != 10) & (seg != 13)).sum(), 0), int(row["slen"])))


def anchor_queries(data, rows, anchors):
    """(row, s, e): whole records around each anchor and windows that start at, end at or cross it"""
    boff = rows["boff"].astype(np.int64)
    q = []
    for at in anchors:
        r = int(np.searchsorted(boff, at, side="right")) - 1
        for rr in range(max(r - 1, 0), min(r + 2, len(rows))):
            sl = int(rows["slen"][rr])
            if sl:
                q.append((rr, 0, sl))
        if r < 0:
            continue
        sl = int(rows["slen"][r])
        p = seq_index(data, rows[r], at)
        for s, e in ((p - 6, p), (p, p + 6), (p - 9, p + 9), (p - 1, p + 1), (p, p + 1), (0, p), (p, sl)):
            s, e = max(s, 0), min(e, sl)
            if e > s:
                q.append((r, s, e))
    return np.array(q, dtype=np.int64).reshape(-1, 3)


def check_fasta(eng, data, anchors):
    exp, total, no_header = fxo.fasta_scan(data)
    f = eng.stage_bytes(data)
    rows, st, drows = eng.fasta_scan(f, keep_device_rows=True)
    assert not no_header
    assert_rows_equal(rows, exp)
    assert (st["n_rows"], st["total_len"]) == (len(exp), total)
    # extraction near the anchors, every flag combination, with and without the counts
    q = anchor_queries(data, exp, anchors)
    rid, s, e = np.repeat(q[:, 0], 8), np.repeat(q[:, 1], 8), np.repeat(q[:, 2], 8)
    fl = np.tile(np.array(FLAGS, np.int32), len(q))
    eo, eoff, eacgt = fxo.subseq_batch(data, exp, rid, s, e, fl, want_acgt=True)
    for want_acgt in (True, False):
        out, off, acgt = eng.extract(f, drows, rid, s, e, fl, want_acgt=want_acgt)
        assert np.array_equal(off, eoff)
        bad = np.nonzero(out != eo)[0]
        if bad.size:
            i = int(np.searchsorted(eoff, bad[0], side="right")) - 1
            raise AssertionError("query %d (row %d [%d, %d) flags %d, acgt %s): got %r expected %r" % (
                i, rid[i], s[i], e[i], fl[i], want_acgt, out[eoff[i]:eoff[i + 1]].tobytes(), eo[eoff[i]:eoff[i + 1]].tobytes()))
        if want_acgt:
            assert np.array_equal(acgt, eacgt)
    for i in range(0, rid.size, 7):
        assert eng.extract_one(f, drows, int(rid[i]), int(s[i]), int(e[i]), int(fl[i])) == eo[eoff[i]:eoff[i + 1]].tobytes()
    # full-index composition
    comp, tot = eng.fasta_composition(f, drows)
    want, want_tot = E.composition(data, exp)
    assert [tuple(int(x) for x in r) for r in comp] == want and np.array_equal(tot, want_tot)
    # search over every record, both strands; with one mismatch on the smaller inputs
    # search, both strands: every record; on the larger inputs the whole records next to the anchors
    if len(data) < SMALL:
        qr, qs, qe = None, None, None
        n = len(exp)
        hays = SL.haystacks(data, exp, np.arange(n), np.zeros(n, np.int64), exp["slen"])
        got = hit_list(eng.search_approx(f, drows, None, None, None, 0, APPROX, 1, BOTH), approx=True)
        assert got == AP.expected_hits(hays, APPROX, 1, 3)
    else:
        qr = np.unique(q[:, 0])
        qs, qe = np.zeros(qr.size, np.int64), exp["slen"][qr].astype(np.int64)
        hays = SL.haystacks(data, exp, qr, qs, qe)
    for pat in PATTERNS:
        assert hit_list(eng.search(f, drows, qr, qs, qe, 0, pat, BOTH)) == SL.expected_hits(hays, pat, 3)
    # split-phase scan, one shard edge at the header line at / after the first anchor and one byte either side of it;
    # then the same at any line (the shard infos)
    cuts = sorted({shard.split_point_bytes(data, a + d, True) for a in anchors[:1] for d in (-1, 0, 1)} - {0, len(data)})
    res = emulate_sharded(eng, data, [0] + cuts + [len(data)], 0)
    assert_rows_equal(np.concatenate([r[0] for r in res]), exp)
    assert sum(r[1]["total_len"] for r in res) == total
    pts = [0] + sorted({shard.split_point_bytes(data, a + d, False) for a in anchors[:1] for d in (-1, 0, 1)}
                       - {0, len(data)}) + [len(data)]
    infos = emulate_sharded(eng, data, pts, 0)[0][2]
    for r in range(len(pts) - 1):
        nl, end, offs, lens = shard_info_expected(data[pts[r]:pts[r + 1]], pts[r])
        assert (int(infos[r]["n_lines"]), int(infos[r]["end_position"])) == (nl, end), r
        assert infos[r]["edge_off"][:len(offs)].tolist() == offs and infos[r]["edge_len"][:len(lens)].tolist() == lens, r
    f.free()
    drows.free()
    # BGZF with a member edge at every anchor
    z, nm = bgzf_at(data, anchors)
    g = eng.stage_bgzf(np.frombuffer(z, np.uint8))
    assert g.n_members in (nm, nm + 1) and g.download().tobytes() == data
    rows_z, st_z = eng.fasta_scan(g)
    assert_rows_equal(rows_z, exp)
    g.free()


def check_fastq(eng, data, anchors):
    exp, size, nlines = fxo.fastq_scan(data)
    f = eng.stage_bytes(data)
    d_rows, st = eng.fastq_scan_dev(f)
    assert (st["n_lines"], st["total_len"], st["n_rows"]) == (nlines, size, len(exp))
    n = len(exp)
    tail = 1 if nlines % 4 else 0
    rows = np.zeros(n + tail, dtype=_cabi.FASTQ_ROW)
    _cabi.check(_cabi.lib().fxg_rows_download(eng.ctx, d_rows, n + tail, _cabi.FASTQ_ROW.itemsize, rows.ctypes.data))
    assert_rows_equal(rows[:n], exp)
    drows = eng.upload_rows(rows)
    # statistics: the reference's line loop, a trailing partial record's sequence line included
    m = eng.fastq_stats(f, drows, n, trailing_seq=nlines % 4 >= 2)
    want = E.fastq_stats(data)
    assert {k: m[k] for k in want} == want
    # every read's bytes, both strands, and read search
    dr = eng.upload_rows(exp)
    hays = [data[int(r["soff"]):int(r["soff"]) + int(r["rlen"])] for r in exp]          # Read.seq: rlen bytes at soff
    for i in range(0, n, max(1, n // 50)):
        assert fxo.read_fetch(data, exp[i])[0] == hays[i]
    seq, qual, off = eng.reads(f, dr, np.arange(n), rlens=exp["rlen"])
    assert seq.tobytes() == b"".join(hays)
    assert qual.tobytes() == b"".join(data[int(r["qoff"]):int(r["qoff"]) + int(r["rlen"])] for r in exp)
    for pat in PATTERNS:
        assert hit_list(eng.search_reads(f, dr, pat, BOTH)) == SL.expected_hits(hays, pat, 3)
    if len(data) < SMALL:
        got = hit_list(eng.search_reads_approx(f, dr, APPROX, 1, BOTH), approx=True)
        assert got == AP.expected_hits(hays, APPROX, 1, 3)
    # split-phase scan, one shard edge at the line start at / after the first anchor and one byte either side of it
    cuts = sorted({shard.split_point_bytes(data, a + d, False) for a in anchors[:1] for d in (-1, 0, 1)} - {0, len(data)})
    res = emulate_sharded(eng, data, [0] + cuts + [len(data)], 1)
    assert_rows_equal(np.concatenate([r[0] for r in res]), exp)
    assert sum(r[1]["n_lines"] for r in res) == nlines and sum(r[1]["total_len"] for r in res) == size
    f.free()
    drows.free()
    dr.free()
    z, nm = bgzf_at(data, anchors)
    g = eng.stage_bgzf(np.frombuffer(z, np.uint8))
    assert g.n_members in (nm, nm + 1) and g.download().tobytes() == data
    rows_z, st_z = eng.fastq_scan(g)
    assert_rows_equal(rows_z, exp)
    assert (st_z["n_lines"], st_z["total_len"]) == (nlines, size)
    g.free()


@pytest.mark.parametrize("layout", sorted(E.layouts()))
def test_edge_layout(eng, layout):
    data, anchors, p = E.build(layout)
    (check_fasta if p.kind == "fasta" else check_fastq)(eng, data, anchors)


@pytest.mark.parametrize("key", sorted(E.CATALOGUE))
def test_catalogue_small_file(eng, key):
    """each pattern on its own, inside one region"""
    p = E.CATALOGUE[key]
    data = E.small_file(p)
    at = len(data) - len(p.data) + p.anchor if p.tail else data.index(p.data) + p.anchor
    (check_fasta if p.kind == "fasta" else check_fastq)(eng, data, [at])


def test_slice_short_of_kept_bytes(eng):
    """a norm=1 record whose last line (21 bases) is longer than its first (20): the slice formula maps the last bases
    onto the line's '\\n', so the covering byte range holds fewer kept bytes than the slice asks for and the rest is
    zero-filled, as in the oracle (SURVEY Q3) -- the strip path once took the kept byte after the range, here the next
    header's '>'"""
    data = b">a\n" + E.S[:20] + b"\n" + E.S[:22] + b"\n>b\nACGT\n"
    exp, _, _ = fxo.fasta_scan(data)
    assert int(exp["norm"][0]) == 1 and int(exp["slen"][0]) == 42
    f = eng.stage_bytes(data)
    rows, st, drows = eng.fasta_scan(f, keep_device_rows=True)
    assert_rows_equal(rows, exp)
    q = [(40, 42, 0), (41, 42, 0), (41, 42, 6), (40, 42, 7), (39, 42, 0), (0, 42, 0)]
    rid, s, e, fl = [0] * len(q), [x[0] for x in q], [x[1] for x in q], [x[2] for x in q]
    eo, eoff, eacgt = fxo.subseq_batch(data, exp, rid, s, e, fl, want_acgt=True)
    assert eo[eoff[0]:eoff[1]].tobytes() == b"T\0"
    out, off, acgt = eng.extract(f, drows, rid, s, e, fl, want_acgt=True)
    assert np.array_equal(off, eoff) and out.tobytes() == eo.tobytes() and np.array_equal(acgt, eacgt)
    for i in range(len(q)):
        assert eng.extract_one(f, drows, 0, s[i], e[i], fl[i]) == eo[eoff[i]:eoff[i + 1]].tobytes()
    drows.free()
    f.free()
