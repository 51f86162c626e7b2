#!/usr/bin/env python3
"""Time pattern search (K8) on the GPU, after verifying what it returns.

    python tools/time_search.py [--steps 10] [--warmup 2] [--records 1000000] [--big-mb 250] [--reads 126000000]
                                [--sections locate,search,reads,approx] [--profile] [--out FILE]

Inputs are generated in HBM with fxg_synth_fasta_dev / fxg_synth_fastq_dev:
    c2   the bench's C2 shape: 1 M FASTA records of U[9000, 11000] bp at 80 columns (~10.2 GB)
    big  one record of --big-mb million bases at 80 columns
    c4   the C4 shape: --reads FASTQ reads of 150 bp (~41.5 GB), scanned with fastq_scan

Timed (CUDA events on the search's stream around `steps` consecutive calls, each of which ends in a host
synchronisation, divided by `steps`):
    locate    every occurrence in every C2 record (what Fasta.locate runs) of a rare 12-mer and of GAATTC, on "+" and on
              "both"; GB/s is file bytes over call time, and its fraction of the H100 SXM's 3.35 TB/s data-sheet figure
    search    Sequence.search's call (first hit of one query) on the big record, against the path it replaces: extract
              the record to the host, decode it, str.find
    reads     every occurrence in every C4 read (what Fastq.locate runs) of the same two patterns on "+" and "both",
              alternating in the same call with the stand-in route it replaces: one-line FASTA rows over the same
              reads through fxg_search_host.  fraction_of_byte_floor: the time to move the 32-byte sectors covering
              every read's sequence plus 32 B per row at 3.35 TB/s, over the call time.  --profile: instead of the
              timings, torch.profiler device time of the new kernels (plan, count, emit)
    approx    the search with mismatches (what Fasta.locate_approx and Fastq.locate_approx run) of the rare 12-mer at
              k = 1, 2, 3 on "+" and "both", on C2 and on C4, alternating in the same call with the exact search of the
              same pattern; ratio_to_exact is its time over the exact search's.  --profile: instead of the timings,
              torch.profiler device time of the count and emit kernels and of the hit copy for each k on "+"

Approx: every reported hit's window (through fxg_extract_host on C2, fxg_reads_host on C4) has the reported number of
mismatches, at most k, against the pattern or its reverse complement; the per-record hit counts of the first 2,000 C2
records and of the first 200,000 C4 reads equal those of numpy windows over the oracle's haystacks of the same bytes.

Reads: every reported hit's window, fetched with fxg_reads_host, equals the pattern (or its reverse complement), and
the per-read hit counts of the first 200,000 reads equal host bytes.find counts on those reads' bytes.

Before any time is printed: every reported C2 hit's window, extracted with fxg_extract_host, equals the pattern (or its
reverse complement on the minus strand), and the per-record hit counts of the first 20,000 records equal those found in
the oracle's haystacks of the same bytes.  The GPU's name, power limit and maximum SM clock are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35
RARE = b"ACGTTGCATGCA"
ECORI = b"GAATTC"
N_ORACLE = 20000
N_ORACLE_READS = 200000
N_ORACLE_APPROX = 2000


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as ex:                                     # reported, never guessed
        return {"error": str(ex)}


def make_fasta(eng, lengths, width=80, seed=20240601):
    from pyfastx_b200 import _cabi, synth
    n = lengths.size
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(synth.fasta_record_sizes(lengths, width=width), out=off[1:])
    f = eng.alloc_file(int(off[-1]))
    dl, do = eng.upload_rows(lengths), eng.upload_rows(off)
    _cabi.check(_cabi.lib().fxg_synth_fasta_dev(eng.ctx, seed, dl.devptr, do.devptr, n, 0, width, f.devptr))
    eng.sync()
    dl.free(); do.free()
    return f, off


def timed(stream, steps, fn):
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(steps):
        fn()
    ev1.record(stream)
    ev1.synchronize()
    return ev0.elapsed_time(ev1) / steps


def verify_c2(eng, f, off, drows, rows, pat, hits):
    """hit windows through the extraction kernel; per-record counts of the first records against the oracle"""
    from oracle import fxo
    from pyfastx_b200 import _cabi
    lut = fxo.complement_lut()
    rc = bytes(lut[np.frombuffer(pat, np.uint8)][::-1])
    m = len(pat)
    q, st, mi = hits["query"], hits["start"], hits["minus"].astype(bool)
    if q.size:
        out, _, _ = eng.extract(f, drows, q, st, st + m, np.zeros(q.size, np.int32))
        win = out.reshape(-1, m)
        want = np.where(mi[:, None], np.frombuffer(rc, np.uint8)[None, :], np.frombuffer(pat, np.uint8)[None, :])
        assert np.array_equal(win, want), "a reported hit's window differs from the pattern"
    n = min(N_ORACLE, len(rows))
    head = f.download(0, int(off[n]))
    orows, _, _ = fxo.fasta_scan(head)
    assert len(orows) == n
    hay, hoff, _ = fxo.subseq_batch(head, orows, np.arange(n), np.zeros(n, np.int64), orows["slen"], np.zeros(n, np.int32))
    hb = hay.tobytes()
    exp = np.zeros((n, 2), dtype=np.int64)
    for i in range(n):
        h = hb[hoff[i]:hoff[i + 1]]
        for s, p in ((0, pat), (1, rc)):
            k = h.find(p)
            while k >= 0:
                exp[i, s] += 1
                k = h.find(p, k + 1)
    sel = q < n
    got = np.zeros((n, 2), dtype=np.int64)
    np.add.at(got, (q[sel], mi[sel].astype(np.int64)), 1)
    assert np.array_equal(got, exp), "hit counts of the first records differ from the oracle"
    return int(exp.sum())


def digits_upto(i):
    total, lo, d = 0, 1, 1
    while lo <= i:
        hi = lo * 10 - 1
        total += (min(i, hi) - lo + 1) * d
        lo *= 10
        d += 1
    return total


def verify_reads(eng, f, rows, pat, hits):
    """hit windows through fxg_reads_host; per-read counts of the first reads against host bytes.find"""
    from oracle import fxo
    lut = fxo.complement_lut()
    rc = bytes(lut[np.frombuffer(pat, np.uint8)][::-1])
    m = len(pat)
    q, st, mi = hits["query"], hits["start"], hits["minus"].astype(bool)
    if q.size:
        win, _ = eng.gather_ranges(f, rows["soff"][q] + st, np.full(q.size, m, np.int64))
        want = np.where(mi[:, None], np.frombuffer(rc, np.uint8)[None, :], np.frombuffer(pat, np.uint8)[None, :])
        assert np.array_equal(win.reshape(-1, m), want), "a reported hit's window differs from the pattern"
    n = min(N_ORACLE_READS, len(rows))
    hb = f.download(0, int(rows["qoff"][n - 1] + rows["rlen"][n - 1] + 1)).tobytes()
    orows, _, _ = fxo.fastq_scan(hb)
    assert len(orows) == n and np.array_equal(orows["soff"], rows["soff"][:n])
    exp = np.zeros((n, 2), dtype=np.int64)
    for i in range(n):
        s = int(orows["soff"][i])
        h = hb[s:s + int(orows["rlen"][i])]
        for k, p in ((0, pat), (1, rc)):
            j = h.find(p)
            while j >= 0:
                exp[i, k] += 1
                j = h.find(p, j + 1)
    sel = q < n
    got = np.zeros((n, 2), dtype=np.int64)
    np.add.at(got, (q[sel], mi[sel].astype(np.int64)), 1)
    assert np.array_equal(got, exp), "hit counts of the first reads differ from host bytes.find"
    return int(exp.sum())


def make_fastq(eng, n):
    """C4-shaped reads generated in HBM and scanned: (file, rows, device rows)"""
    from pyfastx_b200 import _cabi
    f = eng.alloc_file(n * (5 + 11 + 1 + 150 + 1 + 2 + 150 + 1) + digits_upto(n))
    _cabi.check(_cabi.lib().fxg_synth_fastq_dev(eng.ctx, 20240602, n, 0, 150, None, f.devptr))
    eng.sync()
    rows, st, drows = eng.fastq_scan(f, keep_device_rows=True)
    assert len(rows) == n
    return f, rows, st, drows


def window_counts(hay, pat):
    """mismatches of every window of hay (uint8) against pat (uint8); rows of a 2-d hay are haystacks of their own"""
    from numpy.lib.stride_tricks import sliding_window_view
    return (sliding_window_view(hay, pat.size, axis=-1) != pat).sum(axis=-1)


def verify_approx(windows, hay_counts, pat, k, hits, n_first):
    """windows: the hits' windows (n_hits x m); hay_counts(p): per-window mismatch counts of the first n_first haystacks
    against p, as a list of arrays -> number of hits checked against the oracle"""
    from oracle import fxo
    p = np.frombuffer(pat, np.uint8)
    rc = fxo.complement_lut()[p][::-1]
    q, mi, mm = hits["query"], hits["minus"].astype(bool), hits["mismatches"]
    if q.size:
        got = (windows != np.where(mi[:, None], rc[None, :], p[None, :])).sum(axis=1)
        assert np.array_equal(got, mm) and int(mm.max()) <= k, "a reported hit's window has another mismatch count"
    exp = np.zeros((n_first, 2), dtype=np.int64)
    for s, pp in ((0, p), (1, rc)):
        exp[:, s] = [int((c <= k).sum()) for c in hay_counts(pp)]
    sel = q < n_first
    got = np.zeros((n_first, 2), dtype=np.int64)
    np.add.at(got, (q[sel], mi[sel].astype(np.int64)), 1)
    assert np.array_equal(got, exp), "hit counts of the first haystacks differ from numpy windows over the oracle's"
    return int(exp.sum())


def section_approx(a, eng, stream, res):
    """locate_approx of the rare 12-mer on C2 and C4, alternating with the exact search of the same pattern"""
    import torch
    from oracle import fxo
    from pyfastx_b200 import _cabi, synth
    both = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS
    out = res["approx"] = {"pattern": RARE.decode()}
    for shape in ("c2", "c4"):
        _cabi.lib().fxg_pool_trim()
        if shape == "c2":
            lengths = synth.fasta_lengths(a.records, 20240601, 9000, 11000)
            f, off = make_fasta(eng, lengths)
            rows, st, drows = eng.fasta_scan(f, keep_device_rows=True)
            n_first = min(N_ORACLE_APPROX, len(rows))
            head = f.download(0, int(off[n_first]))
            orows, _, _ = fxo.fasta_scan(head)
            hay, hoff, _ = fxo.subseq_batch(head, orows, np.arange(n_first), np.zeros(n_first, np.int64), orows["slen"],
                                            np.zeros(n_first, np.int32))
            hays = [hay[hoff[i]:hoff[i + 1]] for i in range(n_first)]
            hay_counts = lambda p: [window_counts(h, p) for h in hays]
            exact = lambda mask: eng.search(f, drows, None, None, None, 0, RARE, mask)
            approx = lambda k, mask: eng.search_approx(f, drows, None, None, None, 0, RARE, k, mask)
            def windows(h):
                w, _, _ = eng.extract(f, drows, h["query"], h["start"], h["start"] + len(RARE), np.zeros(h.size, np.int32))
                return w.reshape(-1, len(RARE))
        else:
            f, rows, st, drows = make_fastq(eng, a.reads)
            n_first = min(N_ORACLE_READS, len(rows))
            hb = f.download(0, int(rows["qoff"][n_first - 1] + rows["rlen"][n_first - 1] + 1))
            orows, _, _ = fxo.fastq_scan(hb.tobytes())
            assert len(orows) == n_first and np.all(orows["rlen"] == 150)
            reads = hb[orows["soff"][:, None] + np.arange(150)[None, :]]
            hay_counts = lambda p: list(window_counts(reads, p))
            exact = lambda mask: eng.search_reads(f, drows, RARE, mask)
            approx = lambda k, mask: eng.search_reads_approx(f, drows, RARE, k, mask)
            def windows(h):
                w, _ = eng.gather_ranges(f, rows["soff"][h["query"]] + h["start"], np.full(h.size, len(RARE), np.int64))
                return w.reshape(-1, len(RARE))
        o = out[shape] = {"file_gb": f.size / 1e9, "haystacks": len(rows), "bases": int(st["total_len"])}
        for k in (1, 2, 3):
            hits = approx(k, both)
            o["k=%d oracle_checked_hits_first_%d" % (k, n_first)] = verify_approx(windows(hits), hay_counts, RARE, k,
                                                                                 hits, n_first)
            del hits
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            prof_out = o["profile_plus"] = {}
            for k in (1, 2, 3):
                approx(k, _cabi.SEARCH_PLUS)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    approx(k, _cabi.SEARCH_PLUS)
                    torch.cuda.synchronize()
                prof_out["k=%d" % k] = {ev.key: {"calls": ev.count, "device_ms_total": round(ev.device_time_total / 1e3, 3)}
                                        for ev in prof.key_averages() if "approx" in ev.key or "Memcpy DtoH" in ev.key}
        else:
            for k in (1, 2, 3):
                for strand, mask in (("+", _cabi.SEARCH_PLUS), ("both", both)):
                    new, old = (lambda: approx(k, mask)), (lambda: exact(mask))
                    for _ in range(a.warmup):
                        new(); old()
                    n_hits = len(new())
                    tn, to = [], []
                    for _ in range(3):                              # alternating, in the same call
                        tn.append(timed(stream, a.steps, new))
                        to.append(timed(stream, a.steps, old))
                    med, medo = float(np.median(tn)), float(np.median(to))
                    o["k=%d %s" % (k, strand)] = {
                        "hits": n_hits, "ms_median": round(med, 3), "ms_min": round(min(tn), 3), "ms_max": round(max(tn), 3),
                        "exact_ms_median": round(medo, 3), "ratio_to_exact": round(med / medo, 2)}
        drows.free(); f.free()


def section_reads(a, eng, stream, res):
    """Fastq.locate's call on the C4 shape, against the stand-in route: one-line FASTA rows over the same reads
    through fxg_search_host"""
    import torch
    from pyfastx_b200 import _cabi
    n = a.reads
    f, rows, st, drows = make_fastq(eng, n)
    # bytes the search has to read at the least: the 32-byte sectors covering every read's sequence, and its row
    soff, rlen = rows["soff"], rows["rlen"]
    floor = int(((((soff + rlen + 31) >> 5) - (soff >> 5)) * 32).sum()) + 32 * n
    fr = np.zeros(n, dtype=_cabi.FASTA_ROW)
    fr["boff"], fr["blen"], fr["slen"], fr["llen"] = soff, rlen, rlen, rlen + 1
    fr["elen"], fr["norm"] = 1, 1
    fr["pad"][:, 0] = 1
    fdrows = eng.upload_rows(fr)
    del fr
    out = res["reads"] = {"file_gb": f.size / 1e9, "reads": n, "bases": int(st["total_len"]),
                          "byte_floor_gb": floor / 1e9, "byte_floor_ms_at_3.35TBps": round(floor / (HBM_TBS * 1e12) * 1e3, 2)}
    both = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS
    for name, pat in (("rare_12mer", RARE), ("GAATTC", ECORI)):
        hits = eng.search_reads(f, drows, pat, both)
        checked = verify_reads(eng, f, rows, pat, hits)
        stand = eng.search(f, fdrows, None, None, None, 0, pat, both)
        assert np.array_equal(stand, hits), "the stand-in route finds other hits"
        del hits, stand
        for strand, mask in () if a.profile else (("+", _cabi.SEARCH_PLUS), ("both", both)):
            new = lambda: eng.search_reads(f, drows, pat, mask)
            old = lambda: eng.search(f, fdrows, None, None, None, 0, pat, mask)
            for _ in range(a.warmup):
                new(); old()
            n_hits = len(new())
            tn, to = [], []
            for _ in range(3):                                  # alternating, in the same call
                tn.append(timed(stream, a.steps, new))
                to.append(timed(stream, a.steps, old))
            med, medo = float(np.median(tn)), float(np.median(to))
            out["%s %s" % (name, strand)] = {
                "hits": n_hits, "ms_median": round(med, 3), "ms_min": round(min(tn), 3), "ms_max": round(max(tn), 3),
                "file_GBps": round(f.size / (med * 1e-3) / 1e9, 1),
                "fraction_of_byte_floor": round(floor / (HBM_TBS * 1e12) * 1e3 / med, 3),
                "standin_fxg_search_host_ms_median": round(medo, 3), "speedup_vs_standin": round(medo / med, 2),
                "host_checked_hits_first_%d_reads" % N_ORACLE_READS: checked}
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for pat in (RARE, ECORI):
                eng.search_reads(f, drows, pat, _cabi.SEARCH_PLUS)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "search_reads" in ev.key or "Memcpy DtoH" in ev.key:
                kern[ev.key] = {"calls": ev.count, "device_ms_total": round(ev.device_time_total / 1e3, 3)}
        out["profile_rare_then_GAATTC_plus"] = kern
    fdrows.free(); drows.free(); f.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--records", type=int, default=1000000)
    ap.add_argument("--big-mb", type=int, default=250)
    ap.add_argument("--reads", type=int, default=126000000)
    ap.add_argument("--sections", default="locate,search,reads")
    ap.add_argument("--profile", action="store_true", help="reads: torch.profiler device time of each new kernel only")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from pyfastx_b200 import _cabi, engine, synth
    torch.cuda.init()
    eng = engine.Engine(0)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    res = {"gpu": gpu_info(), "device": torch.cuda.get_device_name(0), "locate": {}, "search": {}}
    sections = a.sections.split(",")
    if a.profile:
        if "reads" in sections:
            section_reads(a, eng, stream, res)
        if "approx" in sections:
            section_approx(a, eng, stream, res)
        sections = []

    if "locate" in sections:
        lengths = synth.fasta_lengths(a.records, 20240601, 9000, 11000)
        f, off = make_fasta(eng, lengths)
        rows, st, drows = eng.fasta_scan(f, keep_device_rows=True)
        assert len(rows) == a.records
        res["c2"] = {"file_gb": f.size / 1e9, "records": len(rows), "bases": int(st["total_len"])}
        both = _cabi.SEARCH_PLUS | _cabi.SEARCH_MINUS
        for name, pat in (("rare_12mer", RARE), ("GAATTC", ECORI)):
            hits = eng.search(f, drows, None, None, None, 0, pat, both)
            checked = verify_c2(eng, f, off, drows, rows, pat, hits)
            for strand, mask in (("+", _cabi.SEARCH_PLUS), ("both", both)):
                call = lambda: eng.search(f, drows, None, None, None, 0, pat, mask)
                for _ in range(a.warmup):
                    call()
                n_hits = len(call())
                ms = [timed(stream, a.steps, call) for _ in range(3)]
                med = float(np.median(ms))
                gbs = f.size / (med * 1e-3) / 1e9
                res["locate"]["%s %s" % (name, strand)] = {
                    "hits": n_hits, "ms_median": round(med, 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3),
                    "file_GBps": round(gbs, 1), "fraction_of_3.35TBps": round(gbs / 1e3 / HBM_TBS, 3),
                    "oracle_checked_hits_first_%d_records" % N_ORACLE: checked}
        drows.free(); f.free()

    if "search" in sections:
        big = np.array([a.big_mb * 1000000], dtype=np.int64)
        f, off = make_fasta(eng, big, seed=7)
        rows, _, drows = eng.fasta_scan(f, keep_device_rows=True)
        slen = int(rows["slen"][0])
        rid, s0, e0 = np.array([0]), np.array([0]), np.array([slen])
        seq_tail = eng.extract(f, drows, rid, e0 - 40, e0, np.zeros(1, np.int32))[0].tobytes()
        for name, pat in (("rare_12mer", RARE), ("near_end_20mer", seq_tail[5:25])):
            def gpu_first(strands=_cabi.SEARCH_PLUS):
                h = eng.search(f, drows, rid, s0, e0, 0, pat, strands, first=True)
                return int(h["start"][0]) + 1 if h.size else None
            def host_find():
                k = eng.extract_one(f, drows, 0, 0, slen, 0).decode("latin-1").find(pat.decode())
                return k + 1 if k >= 0 else None
            g, hst = gpu_first(), host_find()
            assert g == hst, (name, g, hst)
            for _ in range(a.warmup):
                gpu_first()
            tg = []
            for _ in range(3):
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    gpu_first()
                tg.append((time.perf_counter() - t0) / a.steps * 1e3)
            th = []
            for _ in range(3):
                t0 = time.perf_counter()
                host_find()
                th.append((time.perf_counter() - t0) * 1e3)
            res["search"][name] = {"record_bases": slen, "answer": g, "gpu_ms_median": round(float(np.median(tg)), 3),
                                   "extract_decode_find_ms_median": round(float(np.median(th)), 1),
                                   "speedup": round(float(np.median(th)) / float(np.median(tg)), 1)}
        drows.free(); f.free()
    if "reads" in sections:
        _cabi.lib().fxg_pool_trim()                         # the freed C2 / big buffers stay pooled: give them back
        section_reads(a, eng, stream, res)
    if "approx" in sections:
        section_approx(a, eng, stream, res)
    s = json.dumps(res, indent=1)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()
