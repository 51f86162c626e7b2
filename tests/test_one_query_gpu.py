"""The one-query getters -- fa[name][s:e].seq / .reverse / .complement / .antisense, fa[name].seq, Sequence[i],
fq[i].seq / .qual / .quali ... -- on every path fxg_extract_one_host / fxg_read_one_host take (tests/onequerylib.py):
the resident service kernel, one launch writing to mapped pinned memory, and one launch writing to a device buffer.

Every answer is compared in full with the oracle (fxo.subseq / fxo.read_fetch) and with the batched extract / reads
of the same query, and the launch counter of the context shows which path served it: a launch-path query adds
exactly one launch, a run of service queries at most one per relaunch of the resident kernel.  Queries of up to
64 KiB take the launch path only with the service off, which the library decides once per process from
FXG_ONE_SERVICE, so those run in a child process started with FXG_ONE_SERVICE=0 (run this file as a script)."""
import ctypes as C
import gc
import hashlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import onequerylib as Q  # noqa: E402
from oracle import fxo  # noqa: E402

pytestmark = pytest.mark.gpu

SVC_RELAUNCHES = 3          # launches a tight run of service queries may add: the resident kernel's (re)starts


def _lib():
    from pyfastx_b200 import _cabi
    return _cabi.lib()


def launches(eng):
    return _lib().fxg_ctx_launch_count(eng.ctx)


def text(b):
    return b.decode("latin-1")


def first_bad(got, want, what):
    bad = [k for k in range(len(want)) if got[k] != want[k]]
    assert not bad, "%d of %d answers differ, first: %r" % (len(bad), len(want), what[bad[0]])


# ---- FASTA ---------------------------------------------------------------------------------------------------------
def check_fasta(eng, fa, fa_up, data, orows, queries, service_on):
    """every (row, s, e, flags) query through its getter on fa (fa_up for UPPER) against the oracle, the batched
    extract as a second witness; the launch counter shows the path.  -> number of queries"""
    names = [fa[i].name for i in range(len(orows))]

    def seq_of(q):
        i, s, e, f = q
        return getattr((fa_up if f & Q.UPPER else fa)[names[i]][s:e], Q.GETTERS[f & Q.RC])

    small = [q for q in queries if q[2] - q[1] <= Q.SVC_LIMIT]
    big = [q for q in queries if q[2] - q[1] > Q.SVC_LIMIT]
    if small:
        want = [text(fxo.subseq(data, orows[i], s, e, f)) for i, s, e, f in small]
        out, off, _ = eng.extract(fa._st.dfile, fa._drows, *zip(*small))
        first_bad([text(out[off[k]:off[k + 1]].tobytes()) for k in range(len(small))], want, small)
        n0 = launches(eng)
        got = [seq_of(q) for q in small]
        n = launches(eng) - n0
        first_bad(got, want, small)
        if service_on:
            assert n <= SVC_RELAUNCHES, "%d launches for %d service queries" % (n, len(small))
        else:
            assert n == len(small), "%d launches for %d launch-path queries" % (n, len(small))
    for q in big:
        i, s, e, f = q
        want = text(fxo.subseq(data, orows[i], s, e, f))
        out, _, _ = eng.extract(fa._st.dfile, fa._drows, [i], [s], [e], [f])
        assert text(out.tobytes()) == want, ("batched", q)
        n0 = launches(eng)
        got = seq_of(q)
        assert launches(eng) - n0 == 1, ("not one launch", q)
        assert got == want, q
    return len(queries)


# ---- FASTQ ---------------------------------------------------------------------------------------------------------
READ_GETTERS = (("seq", 0, 0), ("qual", 1, 0), ("reverse", 0, Q.REVERSE), ("complement", 0, Q.COMPLEMENT),
                ("antisense", 0, Q.RC), ("quali", 1, 0))


def check_reads(eng, fq, data, orows, ids, service_on):
    """.seq .qual .reverse .complement .antisense .quali of every read in ids against the oracle and reads_many, and
    Engine.read_one of the sequence and the quality under all eight upper / reverse / complement combinations against
    the oracle and the batched reads with the same flags.  -> number of getter calls"""
    ids = list(ids)
    seq, qual, off = fq.reads_many(ids)
    aseq, _, aoff = fq.reads_many(ids, want_qual=False, strand_minus=True)
    calls = []                                       # (read, getter name, expected)
    for k, i in enumerate(ids):
        es, eq = fxo.read_fetch(data, orows[i])
        assert seq[off[k]:off[k + 1]].tobytes() == es and qual[off[k]:off[k + 1]].tobytes() == eq, i
        assert aseq[aoff[k]:aoff[k + 1]].tobytes() == Q.transform(es, Q.RC), i
        for name, which, f in READ_GETTERS:
            want = Q.read_expected(data, orows[i], which, f)
            calls.append((i, name, [b - 33 for b in want] if name == "quali" else text(want)))
    small = [c for c in calls if int(orows["rlen"][c[0]]) <= Q.SVC_LIMIT]
    big = [c for c in calls if int(orows["rlen"][c[0]]) > Q.SVC_LIMIT]
    if small:
        n0 = launches(eng)
        got = [getattr(fq[i], name) for i, name, _ in small]
        n = launches(eng) - n0
        first_bad(got, [c[2] for c in small], [c[:2] for c in small])
        assert (n <= SVC_RELAUNCHES) if service_on else (n == len(small)), (n, len(small))
    for i, name, want in big:
        n0 = launches(eng)
        got = getattr(fq[i], name)
        assert launches(eng) - n0 == 1, ("not one launch", i, name)
        assert got == want, (i, name)
    # engine level: every flag combination on the sequence and on the quality line
    dfile, drows = fq._st.dfile, fq._drows
    for f in range(8):
        bs, bq, boff = eng.reads(dfile, drows, ids, flags=f, rlens=orows["rlen"][ids])
        for k, i in enumerate(ids):
            rlen = int(orows["rlen"][i])
            for which, batch in ((0, bs), (1, bq)):
                want = Q.read_expected(data, orows[i], which, f)
                assert batch[boff[k]:boff[k + 1]].tobytes() == want, ("batched", i, which, f)
                n0 = launches(eng)
                got = eng.read_one(dfile, drows, i, rlen, which=which, flags=f)
                n = launches(eng) - n0
                assert got == want, ("read_one", i, which, f)
                assert n == 1 if (rlen > Q.SVC_LIMIT or not service_on) else n <= 1, ("launches", i, which, f, n)
    return len(calls)


# ---- fixtures ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eng():
    from pyfastx_b200 import engine
    return engine.get_engine(0)


@pytest.fixture(scope="module")
def fasta_set(eng, tmp_path_factory):
    import pyfastx_b200 as pyfastx
    data, layouts = Q.fasta_layouts(eng.sm_count)
    path = str(tmp_path_factory.mktemp("one_fa") / "layouts.fa")
    with open(path, "wb") as fh:
        fh.write(data)
    orows, _, _ = fxo.fasta_scan(data)
    fa = pyfastx.Fasta(path)
    fa_up = pyfastx.Fasta(path, uppercase=True)
    return dict(path=path, data=data, layouts=layouts, orows=orows, fa=fa, fa_up=fa_up)


def _fastq(tmp_path_factory, eol, trailing, seed):
    import pyfastx_b200 as pyfastx
    data = Q.fastq_file(Q.FASTQ_LENGTHS, eol=eol, trailing=trailing, seed=seed)
    path = str(tmp_path_factory.mktemp("one_fq") / "reads.fq")
    with open(path, "wb") as fh:
        fh.write(data)
    orows, _, _ = fxo.fastq_scan(data)
    return dict(path=path, data=data, orows=orows, fq=pyfastx.Fastq(path))


@pytest.fixture(scope="module")
def fastq_sets(tmp_path_factory):
    """LF with the last read unterminated, and CRLF"""
    return {"lf": _fastq(tmp_path_factory, b"\n", False, 2), "crlf": _fastq(tmp_path_factory, b"\r\n", True, 3)}


# ---- tests ---------------------------------------------------------------------------------------------------------
def test_layout_rows(fasta_set, fastq_sets):
    """the scan gives each record the intended layout: norm and the uniform-line flag (pad[0] & 1)"""
    fa, orows = fasta_set["fa"], fasta_set["orows"]
    for f in ("boff", "blen", "slen", "llen", "elen", "norm", "dlen", "nlen", "pad"):
        assert np.array_equal(fa._rows[f], orows[f]), f
    for i, lay in enumerate(fasta_set["layouts"]):
        assert fa[i].name == lay["name"] and len(fa[i]) == lay["slen"]
        assert (int(fa._rows["norm"][i]), int(fa._rows["pad"][i][0]) & 1) == (lay["norm"], lay["uniform"]), lay["name"]
    for s in fastq_sets.values():
        assert [int(x) for x in s["fq"]._rows["rlen"]] == Q.FASTQ_LENGTHS
        for f in ("soff", "qoff", "rlen"):
            assert np.array_equal(s["fq"]._rows[f], s["orows"][f]), f


def test_fasta_getters_every_length_start_and_layout(eng, fasta_set):
    """lengths around the service limit, the 2 KiB pieces, the 1 MiB pinned limit and the piece-growth threshold T,
    at start 0, slen - L and an odd middle offset, through .seq .reverse .complement .antisense of a plain and an
    uppercase object; a ~40 MB slice; queries up to 64 KiB on the service, longer ones one launch each"""
    s = fasta_set
    q = Q.fasta_queries(s["layouts"], s["orows"])
    assert check_fasta(eng, s["fa"], s["fa_up"], s["data"], s["orows"], q, service_on=True) == len(q)


def test_sequence_index_slice_of_slice_and_whole_record(eng, fasta_set):
    """Sequence[i], a slice of a slice, and whole-record fa[name].seq of the 46 MB record (one device-buffer launch)"""
    fa, fa_up, data, orows = fasta_set["fa"], fasta_set["fa_up"], fasta_set["data"], fasta_set["orows"]
    for i, lay in enumerate(fasta_set["layouts"]):
        slen = lay["slen"]
        rec = fa[lay["name"]]
        for k in (0, 1, slen // 2 + 1, slen - 1):
            assert rec[k] == text(fxo.subseq(data, orows[i], k, k + 1)), (lay["name"], k)
            assert fa_up[lay["name"]][k - slen] == text(fxo.subseq(data, orows[i], k, k + 1, Q.UPPER))
        for a, b, c, d in ((3, slen - 5, 70_001, 70_001 + 65_537), (slen // 3, slen, 1, 16_385), (0, slen, 5, slen - 7)):
            d = min(d, b - a)
            sub = rec[a:b][c:d]
            assert (sub.start, len(sub)) == (a + c + 1, d - c)
            assert sub.antisense == text(fxo.subseq(data, orows[i], a + c, a + d, Q.RC)), (lay["name"], a, c, d)
    big = fasta_set["layouts"][0]
    n0 = launches(eng)
    whole = fa[big["name"]].seq
    assert launches(eng) - n0 == 1
    assert whole == text(fxo.subseq(data, orows[0], 0, big["slen"]))
    assert fa_up[0].seq == whole.upper()


def test_wrapped_view_without_padding(eng, fasta_set):
    """the file's last record (no trailing newline) in a view whose capacity is its size rounded up to 16: every
    '+ 32 <= capacity' fast-path check fails and the general path serves the query, on every path"""
    fa, data, orows = fasta_set["fa"], fasta_set["data"], fasta_set["orows"]
    size = len(data)
    view = eng.wrap_file(fa._st.dfile.devptr, size, (size + 15) // 16 * 16)
    i = len(orows) - 1
    slen = int(orows["slen"][i])
    qs = [(i, s, s + n, f) for n in fasta_set["layouts"][i]["lengths"] for s in Q.starts(slen, n)
          for f in (0, Q.RC, Q.UPPER | Q.COMPLEMENT)]
    try:
        for r, s, e, f in qs:
            want = fxo.subseq(data, orows[r], s, e, f)
            assert eng.extract_one(view, fa._drows, r, s, e, f) == want, (s, e, f)
        out, off, _ = eng.extract(view, fa._drows, *zip(*qs))
        for k, (r, s, e, f) in enumerate(qs):
            assert out[off[k]:off[k + 1]].tobytes() == fxo.subseq(data, orows[r], s, e, f), (s, e, f)
    finally:
        view.free()                                      # the view only: a wrapped buffer is not owned


@pytest.mark.parametrize("kind", ["lf", "crlf"])
def test_fastq_getters_every_read_length(eng, fastq_sets, kind):
    """reads of 1 .. 3 MiB: every getter, plus Engine.read_one of sequence and quality under every flag combination"""
    s = fastq_sets[kind]
    ids = range(len(Q.FASTQ_LENGTHS))
    assert check_reads(eng, s["fq"], s["data"], s["orows"], ids, service_on=True) == len(Q.FASTQ_LENGTHS) * 6


def _child_cmd(args):
    cmd = [sys.executable]
    if sys.flags.no_user_site:
        cmd.append("-s")
    return cmd + [os.path.abspath(__file__), "child", json.dumps(args)]


def run_child(args):
    """the service-off half: the same checks on the queries of up to 64 KiB, in a process whose library reads
    FXG_ONE_SERVICE=0 -> a JSON line with the counts"""
    import pyfastx_b200 as pyfastx
    from pyfastx_b200 import engine
    eng = engine.get_engine(0)
    data = open(args["fasta"], "rb").read()
    orows, _, _ = fxo.fasta_scan(data)
    lay = [dict(lengths=[n for n in ls if n <= Q.SVC_LIMIT]) for ls in args["lengths"]]
    fa, fa_up = pyfastx.Fasta(args["fasta"]), pyfastx.Fasta(args["fasta"], uppercase=True)
    nfa = check_fasta(eng, fa, fa_up, data, orows, Q.fasta_queries(lay, orows), service_on=False)
    nfq = 0
    for path in args["fastq"]:
        qd = open(path, "rb").read()
        qrows, _, _ = fxo.fastq_scan(qd)
        ids = [i for i in range(len(qrows)) if int(qrows["rlen"][i]) <= Q.SVC_LIMIT]
        nfq += check_reads(eng, pyfastx.Fastq(path), qd, qrows, ids, service_on=False)
    print(json.dumps({"fasta": nfa, "fastq": nfq}))


def test_service_off_launch_path_in_child(fasta_set, fastq_sets):
    """FXG_ONE_SERVICE=0 (read once per process): queries and reads of up to 64 KiB take extract_one_kernel /
    read_one_kernel, one launch each, with the same answers"""
    args = {"fasta": fasta_set["path"], "lengths": [lay["lengths"] for lay in fasta_set["layouts"]],
            "fastq": [s["path"] for s in fastq_sets.values()]}
    env = dict(os.environ, FXG_ONE_SERVICE="0")
    p = subprocess.run(_child_cmd(args), env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    lay = [dict(lengths=[n for n in x["lengths"] if n <= Q.SVC_LIMIT]) for x in fasta_set["layouts"]]
    n_small_reads = sum(1 for n in Q.FASTQ_LENGTHS if n <= Q.SVC_LIMIT)
    assert got == {"fasta": len(Q.fasta_queries(lay, fasta_set["orows"])), "fastq": 2 * 6 * n_small_reads}


def test_composition_and_gc_on_long_slices(fasta_set):
    """Sequence.composition (fxg_composition_host: batched extract + one-CTA-per-query histogram), gc_content and
    gc_skew on slices of 65537 B, 2^20 + 1 B and ~40 MB, against the oracle's bytes"""
    fa, fa_up, data, orows = fasta_set["fa"], fasta_set["fa_up"], fasta_set["data"], fasta_set["orows"]
    for i, lay in enumerate(fasta_set["layouts"]):
        for n in (65537, (1 << 20) + 1, Q.BIG_SLICE):
            if n > lay["slen"]:
                continue
            s = (lay["slen"] - n) // 2 | 1
            for obj, f in ((fa, 0), (fa_up, Q.UPPER)):
                b = fxo.subseq(data, orows[i], s, s + n, f)
                h = fxo.composition(b)
                sub = obj[lay["name"]][s:s + n]
                assert sub.composition == {chr(c): int(h[c]) for c in range(32, 127) if h[c] > 0}, (lay["name"], n, f)
                a, cc, g, t = (int(h[ord(x)] + h[ord(x.lower())]) for x in "ACGT")
                assert sub.gc_content == fxo.gc_content(a, cc, g, t), (lay["name"], n, f)
                assert sub.gc_skew == fxo.gc_skew(cc, g), (lay["name"], n, f)


# ---- interleaving ---------------------------------------------------------------------------------------------------
def _digest(x):
    return hashlib.blake2b(x.encode("latin-1") if isinstance(x, str) else x, digest_size=16).digest()


def _call(objs, fq, item):
    if item[0] == "fa":
        _, key, i, s, e, f = item
        return getattr(objs[key][i][s:e], Q.GETTERS[f])
    _, i, which, f = item
    return getattr(fq[i], "qual" if which else Q.GETTERS[f])


def _expect(datas, uppers, fqd, fqrows, orows, item):
    if item[0] == "fa":
        _, key, i, s, e, f = item
        return _digest(fxo.subseq(datas[key], orows[key][i], s, e, f | (Q.UPPER if uppers[key] else 0)))
    _, i, which, f = item
    return _digest(Q.read_expected(fqd, fqrows[i], which, f))


def test_interleaved_schedule_pool_handover_and_threads(eng, fasta_set, fastq_sets, tmp_path):
    """~2000 seeded getter calls on one engine that switch between two FASTA files, an uppercase object and a FASTQ
    file and between the service, mapped-launch and device-buffer paths, with sleeps past the service's idle period and
    batched extract / reads_many / locate calls in between; halfway, one file is deleted and a different file of the
    same size (>= 64 MiB) opened: it gets the freed device buffer from the pool, and the answers are its bytes.  Then
    the same schedule again from 4 threads at once."""
    import pyfastx_b200 as pyfastx
    L = _lib()
    qs = fastq_sets["lf"]
    fq, fqd, fqrows = qs["fq"], qs["data"], qs["orows"]
    paths, datas = {}, {}
    for key, seed in (("B", 3), ("C", 5)):
        datas[key], _ = Q.fasta_layouts(eng.sm_count, seed=seed)
        paths[key] = str(tmp_path / ("%s.fa" % key))
        with open(paths[key], "wb") as fh:
            fh.write(datas[key])
    assert len(datas["B"]) == len(datas["C"]) == len(fasta_set["data"]) >= 64 << 20 and datas["B"] != datas["C"]
    objs = {"A": fasta_set["fa"], "Aup": fasta_set["fa_up"], "B": pyfastx.Fasta(paths["B"])}
    data_of = {"A": fasta_set["data"], "Aup": fasta_set["data"], "B": datas["B"]}
    uppers = {"A": False, "Aup": True, "B": False}
    orows = {k: fxo.fasta_scan(d)[0] for k, d in data_of.items()}
    slens = {k: r["slen"] for k, r in orows.items()}
    sched = Q.schedule(2000, {k: (slens[k], uppers[k]) for k in objs}, fqrows["rlen"])
    HALF = len(sched) // 2
    rng = np.random.default_rng(11)
    bq = [(int(i), int(s), int(s) + int(n), 0) for i, s, n in
          ((i, rng.integers(0, slens["A"][i] - 5000), rng.integers(1, 5000)) for i in rng.integers(0, 6, 32))]
    bwant = fxo.subseq_batch(fasta_set["data"], orows["A"], *zip(*bq))
    loc0 = objs["A"].locate("ACGTAC", strand="both")
    assert loc0[0].size > 0

    def interlude():
        out, off, _ = objs["A"].extract(*[np.array(x) for x in list(zip(*bq))[:3]])
        assert np.array_equal(out, bwant[0]) and np.array_equal(off, bwant[1])
        sq, ql, off = fq.reads_many(range(len(fqrows)))
        assert all(sq[off[k]:off[k + 1]].tobytes() == fxo.read_fetch(fqd, fqrows[k])[0] for k in range(len(fqrows)))
        loc = objs["A"].locate("ACGTAC", strand="both")
        assert all(np.array_equal(a, b) for a, b in zip(loc, loc0))

    def run(items, check):
        for k, item in items:
            if k % 250 == 0:
                interlude()
            if k in (300, 1300):
                time.sleep(0.02)                         # past the service kernel's idle period: it leaves, then relaunches
            check(k, _digest(_call(objs, fq, item)))

    def expected(items):
        return {k: _expect(data_of, uppers, fqd, fqrows, orows, item) for k, item in items}

    # serial, with the pool hand-over halfway
    first = list(enumerate(sched[:HALF]))
    want = expected(first)
    bad = []
    run(first, lambda k, d: bad.append(k) if d != want[k] else None)
    L.fxg_pool_trim()
    ptr = objs["B"]._st.dfile.devptr
    del objs["B"]
    gc.collect()
    objs["B"] = pyfastx.Fasta(paths["C"])
    assert objs["B"]._st.dfile.devptr == ptr, "the pool did not hand the freed buffer to the file of the same size"
    data_of["B"] = datas["C"]
    orows["B"] = fxo.fasta_scan(datas["C"])[0]
    second = [(k + HALF, it) for k, it in enumerate(sched[HALF:])]
    want.update(expected(second))
    run(second, lambda k, d: bad.append(k) if d != want[k] else None)
    assert not bad, "%d calls differ, first %r" % (len(bad), sched[bad[0]])

    # the same schedule from 4 threads (the getters release the GIL inside the library)
    items = list(enumerate(sched))
    want = expected(items)
    errors = []

    def worker(part):
        try:
            run(part, lambda k, d: errors.append(k) if d != want[k] else None)
        except Exception as ex:                            # noqa: BLE001 -- reported below
            errors.append(repr(ex))

    th = [threading.Thread(target=worker, args=(items[j::4],)) for j in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors[:5]


# ---- upload ordering (C-ABI) ------------------------------------------------------------------------------------------
def test_upload_completes_before_a_one_query_call(eng):
    """fxg_file_from_host returns with the bytes on the device: a one-query call right after it (served by the
    resident kernel on its own stream) sees the new bytes, not what the pooled buffer held before.  A pageable source
    larger than the 256 MiB pinned staging chunk, then a pinned one (fxg_host_alloc)."""
    from pyfastx_b200 import _cabi
    L = _lib()
    data, frows, qrows = Q.upload_order_data()
    n = len(data)
    r, k = len(frows) - 1, len(qrows) - 1
    s, e = Q.UPLOAD_QUERY                                # a service-path query of the last record
    want = (fxo.subseq(data, frows[r], s, e, Q.RC),) + fxo.read_fetch(data, qrows[k])
    rlen = int(qrows["rlen"][k])
    stale = np.full(n, ord("N"), np.uint8)
    src = np.frombuffer(data, np.uint8)
    pinned = C.c_void_p()
    _cabi.check(L.fxg_host_alloc(n, C.byref(pinned)))
    C.memmove(pinned.value, src.ctypes.data, n)
    got = {}
    try:
        for kind, p in (("pageable", src.ctypes.data), ("pinned", pinned.value)):
            L.fxg_pool_trim()
            h = C.c_void_p()
            _cabi.check(L.fxg_file_from_host(eng.ctx, stale.ctypes.data, n, C.byref(h)))     # what the buffer holds before
            ptr = L.fxg_file_devptr(h)
            d_f, d_q = eng.upload_rows(frows), eng.upload_rows(qrows)
            warm = C.create_string_buffer(16)               # the service kernel is resident
            _cabi.check(L.fxg_extract_one_host(eng.ctx, h, d_f.devptr, len(frows), r, 0, 16, 0, warm, 16))
            assert warm.raw == b"N" * 16
            L.fxg_file_free(h)
            _cabi.check(L.fxg_file_from_host(eng.ctx, p, n, C.byref(h)))
            o1, o2, o3 = C.create_string_buffer(e - s), C.create_string_buffer(rlen), C.create_string_buffer(rlen)
            _cabi.check(L.fxg_extract_one_host(eng.ctx, h, d_f.devptr, len(frows), r, s, e, Q.RC, o1, e - s))
            _cabi.check(L.fxg_read_one_host(eng.ctx, h, d_q.devptr, len(qrows), k, 0, 0, rlen, o2, rlen))
            _cabi.check(L.fxg_read_one_host(eng.ctx, h, d_q.devptr, len(qrows), k, 1, 0, rlen, o3, rlen))
            assert L.fxg_file_devptr(h) == ptr, "the upload did not land in the pooled buffer"
            got[kind] = (o1.raw, o2.raw, o3.raw)
            L.fxg_file_free(h)
            d_f.free()
            d_q.free()
    finally:
        L.fxg_host_free(pinned)
    for kind in ("pageable", "pinned"):
        assert got[kind] == want, "%s source: %s" % (kind, [g == w for g, w in zip(got[kind], want)])


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "child":
        run_child(json.loads(sys.argv[2]))
