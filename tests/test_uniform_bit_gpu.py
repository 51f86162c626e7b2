"""The uniform-lines bit (FASTA row pad[0] & 1) on the GPU, on the layouts of tests/uniformlib.py: every scan entry
point (fxg_fasta_scan, fxg_fasta_build_index_host, the split-phase sharded scan) gives every record the oracle's bit,
a Fasta reopened from its .fxi (ours, or one the reference wrote) gets the same bits back, and every kernel that
trusts the bit -- batched extraction, the one-query service and launch paths, fetch_many, locate, locate_approx and
Sequence.search -- answers like the oracle on every layout record, with windows that cross into, lie inside and end
at the record's last line, and queries long enough to be cut into pieces.

The launch path of the one-query getter serves queries of up to 64 KiB only with FXG_ONE_SERVICE=0, which the library
reads once per process, so that part runs in a child process (run this file as a script)."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import approxlib as AP  # noqa: E402
import goldenlib as G  # noqa: E402
import searchlib as SL  # noqa: E402
import shardlib as S  # noqa: E402
import uniformlib as U  # noqa: E402
from oracle import fxo  # noqa: E402

pytestmark = pytest.mark.gpu

RC = fxo.REVERSE | fxo.COMPLEMENT
FLAGS = (0, RC, fxo.UPPER)
BOTH = 3


def assert_rows_equal(got, exp, what):
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    for f in exp.dtype.names:
        bad = np.nonzero((got[f] != exp[f]).reshape(len(exp), -1).any(axis=1))[0]
        assert bad.size == 0, "%s: field %s differs at rows %s: got %s expected %s" % (
            what, f, bad[:5], got[f][bad[:5]], exp[f][bad[:5]])


def all_layouts():
    """(name, data, recs) of every layout file"""
    out = [(k, v.data, v.recs) for k, v in sorted(U.layouts().items())]
    out += [(lay.name, lay.data, lay.recs) for lay in (U.block_layout(d, v) for d, v in U.block_keys())]
    data, recs, _ = U.shard_layout()
    out.append(("shard", data, recs))
    return out


def rec_index(data, rows, recs):
    names = [n.decode() for n in fxo.fasta_names(data, rows)]
    return [names.index(r.name) for r in recs]


def window_queries(rows, idx, recs):
    rid, s, e = [], [], []
    for i, r in zip(idx, recs):
        for a, b in U.windows(rows[i], r):
            rid.append(i); s.append(a); e.append(b)
    return np.array(rid, np.int64), np.array(s, np.int64), np.array(e, np.int64)


@pytest.fixture(scope="module")
def eng():
    from pyfastx_b200 import engine
    return engine.get_engine(0)


@pytest.fixture(scope="module")
def engs():
    from pyfastx_b200 import engine
    es = [engine.Engine(0) for _ in range(max(U.SHARD_WORLDS))]
    yield es
    for e in es:
        e.close()


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    """every layout written to a file: name -> (path, data, recs)"""
    d = tmp_path_factory.mktemp("uniform_bit")
    out = {}
    for name, data, recs in all_layouts():
        path = str(d / (name + ".fa"))
        with open(path, "wb") as f:
            f.write(data)
        out[name] = (path, data, recs)
    return out


# ---- the bit -------------------------------------------------------------------------------------------------------
def test_scan_entry_points_give_the_oracle_bit(eng, engs, files):
    """fxg_fasta_scan, fxg_fasta_build_index_host and the split-phase scan of 3 ranks: every row, pad included"""
    for name, (_, data, recs) in files.items():
        exp, total, _ = fxo.fasta_scan(data)
        idx = rec_index(data, exp, recs)
        assert [int(exp["pad"][i, 0]) for i in idx] == [int(r.uniform) for r in recs], name
        f = eng.stage_bytes(data)
        try:
            rows, st = eng.fasta_scan(f)
        finally:
            f.free()
        assert_rows_equal(rows, exp, (name, "scan"))
        rows, st = eng.fasta_build_index_host(data)
        assert_rows_equal(rows, exp, (name, "host"))
        from pyfastx_b200 import shard
        pts = shard.fasta_split_points(data, 3)
        res, _ = S.emulate(engs, pts, 0, data=data)
        assert_rows_equal(np.concatenate([p["rows"] for p in res]), exp, (name, "shards"))


@pytest.mark.parametrize("world", U.SHARD_WORLDS)
def test_first_record_of_a_shard(engs, world):
    """every layout record as the first record of a shard (and, with consecutive cuts, the only one)"""
    data, recs, _ = U.shard_layout()
    exp, total, _ = fxo.fasta_scan(data)
    for cuts in U.shard_cuts(world):
        pts = [0] + cuts + [len(data)]
        res, _ = S.emulate(engs, pts, 0, data=data)
        assert_rows_equal(np.concatenate([p["rows"] for p in res]), exp, (world, cuts))
        assert sum(int(p["stats"]["total_len"]) for p in res) == total


def test_reopened_index_gets_the_bits_back(files, tmp_path):
    """a Fasta opened from the .fxi it wrote, and one opened from the index the reference wrote for the same file:
    _verify_loaded_index restores pad from one scan"""
    import pyfastx_b200 as pyfastx
    for name in ("fact_nl", "carry_2k_nl", "dense_nl", "general_facts_nl", "rows01_k1_eof_plus1_crlf_lf", "shard"):
        path, data, _ = files[name]
        exp, _, _ = fxo.fasta_scan(data)
        fa = pyfastx.Fasta(path, index_file=str(tmp_path / (name + ".fxi")))
        assert np.array_equal(fa._rows["pad"], exp["pad"]), name
        del fa
        fb = pyfastx.Fasta(path, index_file=str(tmp_path / (name + ".fxi")))
        assert fb.index_matches_file and np.array_equal(fb._rows["pad"], exp["pad"]), name
    data = gzip.open(os.path.join(G.GOLD, "data", "test.fa.gz")).read()
    path = str(tmp_path / "theirs.fa")
    with open(path, "wb") as f:
        f.write(data)
    G.ref_fxi("test.fa", path + ".fxi")
    exp, _, _ = fxo.fasta_scan(data)
    fc = pyfastx.Fasta(path)
    assert fc.index_matches_file and np.array_equal(fc._rows["pad"], exp["pad"])


# ---- the kernels that trust it -------------------------------------------------------------------------------------
def check_extract(eng, f, drows, data, exp, idx, recs, what):
    """Engine.extract with flags 0, RC, UPPER, with and without A/C/G/T counts; windows of 16 .. 4096 bytes take the
    bulk path on uniform records"""
    rid, s, e = window_queries(exp, idx, recs)
    for fl in FLAGS:
        flags = np.full(rid.size, fl, np.int32)
        eo, eoff, eacgt = fxo.subseq_batch(data, exp, rid, s, e, flags, want_acgt=True)
        for want in (False, True):
            out, off, acgt = eng.extract(f, drows, rid, s, e, flags, want_acgt=want)
            assert np.array_equal(off, eoff), what
            bad = np.flatnonzero(out != eo)
            if bad.size:
                q = int(np.searchsorted(eoff, bad[0], side="right")) - 1
                raise AssertionError("%s: query %d (row %d [%d, %d) flags %d): got %r expected %r" % (
                    what, q, rid[q], s[q], e[q], fl, out[eoff[q]:eoff[q + 1]].tobytes()[:80],
                    eo[eoff[q]:eoff[q + 1]].tobytes()[:80]))
            if want:
                assert np.array_equal(acgt, eacgt), what


def check_extract_one(eng, f, drows, data, exp, idx, recs, what):
    """the one-query getter, windows of more than 2 KiB cut into pieces -> number of queries"""
    rid, s, e = window_queries(exp, idx, recs)
    n = 0
    for fl in (0, RC):
        flags = np.full(rid.size, fl, np.int32)
        eo, eoff, _ = fxo.subseq_batch(data, exp, rid, s, e, flags)
        for q in range(rid.size):
            got = eng.extract_one(f, drows, int(rid[q]), int(s[q]), int(e[q]), fl)
            assert got == eo[eoff[q]:eoff[q + 1]].tobytes(), (what, int(rid[q]), int(s[q]), int(e[q]), fl)
            n += 1
    return n


def check_api(path, data, recs, what):
    """fetch_many, locate, locate_approx and Sequence.search through a Fasta object"""
    import pyfastx_b200 as pyfastx
    fa = pyfastx.Fasta(path, index_file=path + ".fxi")
    exp, _, _ = fxo.fasta_scan(data)
    idx = rec_index(data, exp, recs)
    rid, s, e = window_queries(exp, idx, recs)
    names = [r.name for r in recs]
    by_row = dict(zip(idx, names))
    strands = ["+" if k % 2 else "-" for k in range(rid.size)]
    got = fa.fetch_many([by_row[int(i)] for i in rid], s + 1, e, strands)
    for k in range(rid.size):
        want = fxo.fetch(data, exp[rid[k]], [(int(s[k]) + 1, int(e[k]))], strands[k])
        assert got[k] == want.decode("latin-1"), (what, "fetch_many", int(rid[k]), int(s[k]), int(e[k]), strands[k])
    # whole records: every record of the layouts is longer than one search piece but the short ones of general_facts
    hays = SL.haystacks(data, exp, np.array(idx), np.zeros(len(idx), np.int64), exp["slen"][idx])
    mine = np.zeros(len(exp), bool)
    mine[idx] = True
    pos = {int(i): k for k, i in enumerate(idx)}
    r, st, mi = fa.locate(U.PATTERN, "both")
    keep = mine[r]
    got = sorted((pos[int(a)], int(b), int(c)) for a, b, c in zip(r[keep], st[keep], mi[keep]))
    assert got == SL.expected_hits(hays, U.PATTERN, BOTH), (what, "locate")
    crossing = [h for h in got if h[1] < recs[h[0]].last_start <= h[1] + len(U.PATTERN)]     # a hit up to the last break
    assert crossing or all(r.variant == "empty" for r in recs), what
    r, st, mi, mm = fa.locate_approx(U.PATTERN, 2, "both")
    keep = mine[r]
    got = sorted((pos[int(a)], int(b), int(c), int(d)) for a, b, c, d in zip(r[keep], st[keep], mi[keep], mm[keep]))
    assert got == AP.expected_hits(hays, U.PATTERN, 2, BOTH), (what, "locate_approx")
    pat = U.PATTERN.decode()
    for k, (i, rec) in enumerate(zip(idx, recs)):
        sq = fa[int(i)]
        assert sq.search(pat) == SL.first_position(hays[k], U.PATTERN, False), (what, rec.name)
        assert sq.search(pat, "-") == SL.first_position(hays[k], U.PATTERN, True), (what, rec.name)
        a, slen = max(0, rec.last_start - 3000), int(exp["slen"][i])
        want = SL.first_position(fxo.subseq(data, exp[i], a, slen), U.PATTERN, False)
        assert sq[a:slen].search(pat) == want, (what, rec.name, "slice")
    del fa


@pytest.mark.parametrize("family", list(U.FAMILIES) + ["block", "shard"])
def test_consumers(eng, files, family):
    """extract, the one-query service, fetch_many, locate, locate_approx, Sequence.search on every layout record"""
    names = [n for n in files if n == family or n.startswith(family + "_") or (family == "block" and n.startswith("block"))]
    assert names
    n = 0
    for name in names:
        path, data, recs = files[name]
        exp, _, _ = fxo.fasta_scan(data)
        idx = rec_index(data, exp, recs)
        f = eng.stage_bytes(data)
        drows = eng.upload_rows(exp)
        try:
            check_extract(eng, f, drows, data, exp, idx, recs, name)
            n += check_extract_one(eng, f, drows, data, exp, idx, recs, name)
        finally:
            drows.free()
            f.free()
        check_api(path, data, recs, name)
    assert n > 0


def run_child(args):
    """the launch path (FXG_ONE_SERVICE=0): every layout's windows through extract_one -> JSON counts"""
    from pyfastx_b200 import engine
    eng = engine.get_engine(0)
    n = 0
    for name, data, recs in all_layouts():
        exp, _, _ = fxo.fasta_scan(data)
        idx = rec_index(data, exp, recs)
        f = eng.stage_bytes(data)
        drows = eng.upload_rows(exp)
        try:
            n += check_extract_one(eng, f, drows, data, exp, idx, recs, name)
        finally:
            drows.free()
            f.free()
    print(json.dumps({"queries": n}))


def test_one_query_launch_path_in_child():
    """FXG_ONE_SERVICE=0: the same windows through extract_one_kernel, one launch each"""
    want = 0
    for name, data, recs in all_layouts():
        exp, _, _ = fxo.fasta_scan(data)
        want += 2 * window_queries(exp, rec_index(data, exp, recs), recs)[0].size
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "child", "{}"]
    p = subprocess.run(cmd, env=dict(os.environ, FXG_ONE_SERVICE="0"), cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert json.loads(p.stdout.strip().splitlines()[-1]) == {"queries": want}


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "child":
        run_child(json.loads(sys.argv[2]))
