"""The batched gather (K3/K4/K5, csrc/fxg_extract.cu) past one batch per warp and past 2^21 queries, against the
oracle: every byte, offset and A/C/G/T count of queries laid out at chosen lane positions (gatherlib.lane_queries), of
the three large sets, of fxg_composition_host, of reads at scale and of Fasta.fetch_many.  gatherlib states the inputs,
test_gather_scale_cpu.py that they reach what they aim at."""
import ctypes as C

import numpy as np
import pytest

import gatherlib as G
import pyfastx_b200 as pyfastx
from oracle import fxo
from pyfastx_b200 import _cabi, engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    return engine.get_engine(0)


@pytest.fixture(scope="module")
def mixed(eng):
    data, kinds = G.mixed_fasta()
    exp_rows = fxo.fasta_scan(data)[0]
    f = eng.stage_bytes(data)
    rows, _, drows = eng.fasta_scan(f, keep_device_rows=True)
    yield data, kinds, rows, exp_rows, f, drows
    drows.free()
    f.free()


def _first_bad(got, want, off, what):
    """index of the first query whose bytes differ, or None"""
    bad = np.flatnonzero(got != want)
    if bad.size == 0:
        return None
    return int(np.searchsorted(off, bad[0], side="right") - 1)


def check_extract(data, rows, kinds, q, out, off, acgt, label):
    rid, s, e, fl = q["rid"], q["s"], q["e"], q["flags"]
    want_off = np.concatenate([[0], np.cumsum(np.maximum(e - s, 0))])
    assert np.array_equal(off, want_off), label
    eo, _, eacgt = G.expected(data, rows, rid, s, e, fl, G.formula_rows(kinds))
    uni = (rows["pad"][:, 0] & 1) != 0
    i = _first_bad(out, eo, off, label)
    if i is None and acgt is not None:
        bad = np.flatnonzero((acgt != eacgt).any(axis=1))
        i = int(bad[0]) if bad.size else None
    if i is not None:
        fast, npi = G.bulk_fast(rows, uni, rid[i:i + 1], s[i:i + 1], e[i:i + 1], fl[i:i + 1], off[i:i + 1], 1 << 40)
        pull = G.pull_ok(rows, uni, rid[i:i + 1], s[i:i + 1], e[i:i + 1], fl[i:i + 1], len(data), 1 << 40)
        kind = q["kind"][i] if "kind" in q else "random"
        rk = kinds[rid[i]]["kind"] if 0 <= rid[i] < len(rows) else None
        pytest.fail("%s: query %d kind %s on record %s (%s) s=%d e=%d flags=%d a=%d np=%d path %s: got %r want %r"
                    " acgt %s vs %s" % (label, i, kind, rid[i], rk, s[i], e[i], fl[i], off[i] & 15, npi[0],
                                        G.path_of(kind, fast[0], pull[0], rk), out[off[i]:off[i + 1]][:80].tobytes(),
                                        eo[off[i]:off[i + 1]][:80].tobytes(),
                                        None if acgt is None else acgt[i].tolist(), eacgt[i].tolist()))


@pytest.mark.parametrize("bq", [None, 1, 3, 8, 31, 32])
def test_mixed_batches(eng, mixed, monkeypatch, bq):
    """lane_queries at each forced batch width (unset: the width-32 set, which the default runs at width 32), with and
    without the A/C/G/T counts; and the scan layout every record was built for"""
    data, kinds, rows, exp_rows, f, drows = mixed
    for k, r in zip(kinds, rows):
        assert (int(r["norm"]), bool(r["pad"][0] & 1)) == (k["norm"], k["uniform"]), k["name"]
    if bq is not None:
        monkeypatch.setenv("FXG_BK_BQ", str(bq))
    q = G.lane_queries(data, kinds, rows, bq or 32)
    for want in (False, True):
        out, off, acgt = eng.extract(f, drows, q["rid"], q["s"], q["e"], q["flags"], want_acgt=want)
        check_extract(data, rows, kinds, q, out, off, acgt, "bq=%s acgt=%s" % (bq, want))


@pytest.mark.parametrize("nq", G.LARGE_SIZES)
def test_past_2_21_queries(eng, mixed, nq):
    """2^21, 2^21 + 1 and 2 * 2^21 + 2048 + 7 queries: one, two and three chunks of ps_scan_sums; the first two also
    through fxg_extract_plan_dev + fxg_extract_dev on torch device tensors, as bench.py calls them"""
    import torch
    data, kinds, rows, exp_rows, f, drows = mixed
    q = G.large_queries(rows, nq)
    out, off, acgt = eng.extract(f, drows, q["rid"], q["s"], q["e"], q["flags"], want_acgt=True)
    check_extract(data, rows, kinds, q, out, off, acgt, "extract nq=%d" % nq)
    if nq == G.LARGE_SIZES[-1]:
        return
    L = _cabi.lib()
    d_rid, d_s, d_e = (torch.from_numpy(q[k]).cuda() for k in ("rid", "s", "e"))
    d_fl = torch.from_numpy(q["flags"]).cuda()
    d_off = torch.full((nq + 1,), -1, dtype=torch.int64, device="cuda")
    d_acgt = torch.full((nq, 4), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    total = C.c_int64(-1)
    _cabi.check(L.fxg_extract_plan_dev(eng.ctx, d_s.data_ptr(), d_e.data_ptr(), nq, d_off.data_ptr(), C.byref(total)))
    assert total.value == int(off[-1])
    d_out = torch.full((total.value + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    _cabi.check(L.fxg_extract_dev(eng.ctx, f.handle, drows.devptr, drows.n_rows, d_rid.data_ptr(), d_s.data_ptr(),
                                  d_e.data_ptr(), d_fl.data_ptr(), nq, d_off.data_ptr(), d_out.data_ptr(),
                                  d_acgt.data_ptr()))
    eng.sync()
    got = d_out.cpu().numpy()
    assert (got[total.value:] == 0xAB).all()
    check_extract(data, rows, kinds, q, got[:total.value], d_off.cpu().numpy(), d_acgt.cpu().numpy(), "dev nq=%d" % nq)


@pytest.fixture(scope="module")
def fastqs(eng):
    out = {}
    for eol, trailing in ((b"\n", True), (b"\r\n", False)):
        data = G.reads_fastq(eol, trailing=trailing)
        f = eng.stage_bytes(data)
        rows, _, drows = eng.fastq_scan(f, keep_device_rows=True)
        assert np.array_equal(rows["rlen"], fxo.fastq_scan(data)[0]["rlen"])
        out[len(eol)] = (data, rows, f, drows)
    yield out
    for data, rows, f, drows in out.values():
        drows.free()
        f.free()


def test_reads_past_2_21(eng, fastqs):
    """2^21 + 1 reads (a second chunk of the offset prefix) through fxg_reads_host and fxg_reads_dev"""
    import torch
    data, rows, f, drows = fastqs[1]
    rng = np.random.default_rng(7)
    nq = (1 << 21) + 1
    small = np.flatnonzero(rows["rlen"] <= 40)
    ids = small[rng.integers(0, small.size, nq)]
    ids[rng.integers(0, nq, 300)] = rng.integers(0, len(rows), 300)
    ids[-1] = len(rows) - 1
    for flags in (0, G.RC):
        es, eq, eoff = G.expect_reads(data, rows, ids, flags)
        seq, qual, off = eng.reads(f, drows, ids, flags=flags, rlens=rows["rlen"][ids])
        assert np.array_equal(off, eoff) and np.array_equal(seq, es) and np.array_equal(qual, eq), flags
    L = _cabi.lib()
    total = int(eoff[-1])
    d_ids = torch.from_numpy(ids).cuda()
    d_off = torch.full((nq + 1,), -1, dtype=torch.int64, device="cuda")
    d_seq = torch.full((total + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    d_qual = torch.full((total + 64,), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    got_total = C.c_int64(-1)
    _cabi.check(L.fxg_reads_dev(eng.ctx, f.handle, drows.devptr, drows.n_rows, d_ids.data_ptr(), nq, G.RC,
                                d_off.data_ptr(), d_seq.data_ptr(), d_qual.data_ptr(), total + 64, C.byref(got_total)))
    eng.sync()
    assert got_total.value == total
    assert np.array_equal(d_off.cpu().numpy(), eoff)
    s, q = d_seq.cpu().numpy(), d_qual.cpu().numpy()
    assert (s[total:] == 0xAB).all() and (q[total:] == 0xAB).all()
    assert np.array_equal(s[:total], es) and np.array_equal(q[:total], eq)


@pytest.mark.parametrize("crlf", [False, True], ids=["lf", "crlf"])
def test_reads_at_scale(eng, fastqs, crlf):
    """60k ids with repeats (reads of 1..600 bytes, 40 of 20k or more, the last read of the file): flags 0, 2, 4, 6 with
    sequence only, quality only and both"""
    data, rows, f, drows = fastqs[2 if crlf else 1]
    rng = np.random.default_rng(11)
    ids = rng.integers(0, len(rows), 60_000)
    ids[:40] = np.flatnonzero(rows["rlen"] >= 20_000)
    ids[-1] = len(rows) - 1
    rng.shuffle(ids)
    assert np.unique(ids).size < ids.size
    for flags in (0, 2, 4, 6):
        es, eq, eoff = G.expect_reads(data, rows, ids, flags)
        for ws, wq in ((True, False), (False, True), (True, True)):
            seq, qual, off = eng.reads(f, drows, ids, flags=flags, want_seq=ws, want_qual=wq, rlens=rows["rlen"][ids])
            assert np.array_equal(off, eoff)
            if ws:
                i = _first_bad(seq, es, off, "seq")
                assert i is None, (flags, i, int(ids[i]), int(rows["rlen"][ids[i]]))
            if wq:
                i = _first_bad(qual, eq, off, "qual")
                assert i is None, (flags, i, int(ids[i]), int(rows["rlen"][ids[i]]))


def test_composition_host(eng, mixed):
    """fxg_composition_host on 30k mixed queries with every flag: a per-query bincount of the oracle's bytes"""
    data, kinds, rows, exp_rows, f, drows = mixed
    q = G.lane_queries(data, kinds, rows, 8)
    n = 30_000
    q = {k: v[:n] for k, v in q.items()}
    assert (np.isin(q["flags"] & 7, range(8))).all() and len(set((q["flags"] & 7).tolist())) == 8
    hist = np.zeros((n, 256), np.int64)
    _cabi.check(_cabi.lib().fxg_composition_host(eng.ctx, f.handle, drows.devptr, drows.n_rows, q["rid"].ctypes.data,
                                                 q["s"].ctypes.data, q["e"].ctypes.data, q["flags"].ctypes.data, n,
                                                 hist.ctypes.data))
    eo, eoff, _ = G.expected(data, rows, q["rid"], q["s"], q["e"], q["flags"], G.formula_rows(kinds))
    qi = np.repeat(np.arange(n), np.diff(eoff))
    want = np.bincount(qi * 256 + eo, minlength=n * 256).reshape(n, 256)
    bad = np.flatnonzero((hist != want).any(axis=1))
    assert bad.size == 0, (int(bad[0]), q["kind"][bad[0]], int(q["rid"][bad[0]]), int(q["s"][bad[0]]),
                           int(q["e"][bad[0]]), int(q["flags"][bad[0]]))


def test_fetch_many(tmp_path, mixed):
    """Fasta.fetch_many on 100k intervals over the mixed file, mixed strands, against the oracle under WHOLE.  On a
    record with uniform lines the kernel indexes with the slice formula (DESIGN.md section 4): on 'bad_crlf', whose one
    CRLF line ends in a letter + '\\n', that is the oracle without WHOLE."""
    data, kinds, rows, exp_rows, f, drows = mixed
    p = tmp_path / "mixed.fa"
    p.write_bytes(data)
    fa = pyfastx.Fasta(str(p))
    rng = np.random.default_rng(3)
    n = 100_000
    rid = rng.integers(0, len(rows), n)
    slen = rows["slen"][rid]
    ln = np.where(rng.random(n) < 0.95, rng.integers(1, 400, n), rng.integers(1024, 3000, n))
    st = 1 + (rng.random(n) * slen).astype(np.int64)                       # 1-based, inclusive
    en = st + ln - 1 + np.where(rng.random(n) < 0.02, 50, 0)               # some past the record's end
    minus = rng.random(n) < 0.5
    names = [kinds[i]["name"] for i in rid]
    got = fa.fetch_many(names, st, en, ["-" if m else "+" for m in minus])
    s0 = np.clip(st - 1, 0, slen)
    e0 = np.clip(en, s0, slen)
    formula = G.formula_rows(kinds)[rid]
    assert formula.sum() > 1000
    flags = (np.where(formula, 0, G.WHOLE) | np.where(minus, G.RC, 0)).astype(np.int32)
    eo, eoff, _ = fxo.subseq_batch(data, exp_rows, rid, s0, e0, flags)
    buf = eo.tobytes().decode("latin-1")
    for i in range(n):
        if got[i] != buf[eoff[i]:eoff[i + 1]]:
            pytest.fail("interval %d on %s [%d, %d] %s: got %r want %r" % (
                i, names[i], st[i], en[i], "-" if minus[i] else "+", got[i][:60], buf[eoff[i]:eoff[i + 1]][:60]))
