#!/usr/bin/env python3
"""Per-kernel time of one index-build scan step (fxg_scan_sharded, one rank), by kernel name, on three seeded inputs
generated in HBM:

    c2        1 M FASTA records of U[9000, 11000] bp at 80 columns (the bench's C2 shape, ~10.2 GB)
    short_fa  FASTA records of U[100, 300] bp at 60 columns, ~2 GB (most regions take the general rows path)
    c4        FASTQ, 150 bp reads, ~10 GB

For each shape: the mean time per step of every kernel (torch.profiler, CUDA activities, in a run of its own), the
step time, and the sha256 of all rows downloaded from the device, pad bytes included.  FXG_LIB_PATH=... runs the same script against another build of
libfxg.so, so that two builds can be compared for time and output identity.

    python tools/time_scan_phases.py [--shapes c2,short_fa,c4] [--steps 10] [--out FILE]

The step time is taken as bench.py takes it: CUDA events on the scan's stream around `steps` consecutive calls, with the
profiler off, divided by `steps`.  Every call ends in a stream synchronise, so the window also holds the host turnaround
between calls (launches, the one device-to-host copy of the totals); the per-kernel table is the device time alone.
Repeat the script with and without FXG_LIB_PATH, alternating, to compare two builds.
"""
import argparse
import hashlib
import json
import os
import sys
from collections import defaultdict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_fasta(eng, L, synth, n, min_len, max_len, width, seed=20240601):
    lengths = synth.fasta_lengths(n, seed, min_len, max_len)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(synth.fasta_record_sizes(lengths, width=width), out=off[1:])
    f = eng.alloc_file(int(off[-1]))
    dl, do = eng.upload_rows(lengths), eng.upload_rows(off)
    from pyfastx_b200 import _cabi
    _cabi.check(L.fxg_synth_fasta_dev(eng.ctx, seed, dl.devptr, do.devptr, n, 0, width, f.devptr))
    eng.sync()
    dl.free(); do.free()
    return f


def make_fastq(eng, L, n, seed=20240602):
    from pyfastx_b200 import _cabi
    nbytes = n * (5 + 11 + 1 + 150 + 1 + 2 + 150 + 1) + sum((min(n, 10 ** (d + 1) - 1) - 10 ** d + 1) * (d + 1)
                                                          for d in range(10) if 10 ** d <= n)
    f = eng.alloc_file(nbytes)
    _cabi.check(L.fxg_synth_fastq_dev(eng.ctx, seed, n, 0, 150, None, f.devptr))
    eng.sync()
    return f


def measure(eng, stream, f, mode, steps, warmup):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        eng.scan_sharded_dev(None, f, mode)
    # output identity: every row, every byte
    rows, st, infos = eng.scan_sharded(None, f, mode)
    digest = hashlib.sha256(rows.tobytes()).hexdigest()
    info_digest = hashlib.sha256(infos.tobytes()).hexdigest()
    # step time, profiler off: CUDA events on the scan's stream around windows of `steps` calls
    ts = []
    for _ in range(3):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        for _ in range(steps):
            eng.scan_sharded_dev(None, f, mode)
        ev1.record(stream)
        ev1.synchronize()
        ts.append(ev0.elapsed_time(ev1) / steps)
    # per-kernel time, in a run of its own
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.scan_sharded_dev(None, f, mode)
        torch.cuda.synchronize()
    per = defaultdict(float)
    cnt = defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time_total > 0:
            name = ev.name
            if name.startswith("Memcpy") or name.startswith("Memset"):
                name = name.split(" ")[0]
            per[name] += ev.device_time_total / 1e3
            cnt[name] += 1
    kernels = {k: {"ms_per_step": round(v / steps, 5), "calls_per_step": cnt[k] / steps}
               for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
    return {"file_gb": f.size / 1e9, "n_rows": int(st["n_rows"]), "total_len": int(st["total_len"]),
            "rows_sha256": digest, "shard_info_sha256": info_digest,
            "step_ms_median": round(float(np.median(ts)), 4), "step_ms_min": round(float(np.min(ts)), 4),  # of 3 windows
            "step_ms_max": round(float(np.max(ts)), 4),
            "kernels_ms_sum": round(sum(v["ms_per_step"] for v in kernels.values()), 5), "kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,short_fa,c4")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from pyfastx_b200 import _cabi, engine, synth
    L = _cabi.lib()
    torch.cuda.init()
    eng = engine.Engine(0)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    out = {"lib": _cabi.LIB_PATH, "device": torch.cuda.get_device_name(0), "shapes": {}}
    for shape in a.shapes.split(","):
        if shape == "c2":
            f, mode = make_fasta(eng, L, synth, 1000000, 9000, 11000, 80), 0
        elif shape == "short_fa":
            f, mode = make_fasta(eng, L, synth, 8500000, 100, 300, 60), 0
        elif shape == "c4":
            f, mode = make_fastq(eng, L, 30000000), 1
        else:
            raise SystemExit("unknown shape %r" % shape)
        out["shapes"][shape] = measure(eng, stream, f, mode, a.steps, a.warmup)
        f.free()
    s = json.dumps(out, indent=1)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(s + "\n")
    print(s)


if __name__ == "__main__":
    main()
