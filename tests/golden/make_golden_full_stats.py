#!/usr/bin/env python3
"""Generate tests/golden/full_stats.json.gz from the UNMODIFIED reference (oracle/_ref build): the full-index
statistics of the statslib inputs small enough for it.

- FASTA (many_records, and tile_sweep with ASCII lines and no 64 MiB record): a digest (statslib.comp_digest) of the
  `comp` table of the .fxi, and the composition / gc_content / gc_skew / type getters.  FASTA inputs with bytes >= 128
  are left out: the reference indexes a 128-entry array with them.
- FASTQ (quality_classes and step_sweep, LF and CRLF, many_reads and the INNER_CR files): the `base` / `meta` rows, the statistics getters
  and encoding_type.  Quality bytes >= 128 stay in: the reference only compares them.

    bash oracle/build_ref.sh && python tests/golden/make_golden_full_stats.py

tests/test_full_stats_cpu.py pins the statslib restatements to these answers."""
import gzip
import json
import os
import shutil
import sqlite3
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import pyfastx  # noqa: E402  (the compiled reference)
import statslib as S  # noqa: E402


def fasta_inputs():
    yield "many_records", S.many_records
    yield "tile_sweep_ascii", lambda: S.tile_sweep(big=0, ascii_only=True)


def fastq_inputs():
    for eol, tag in ((b"\n", "lf"), (b"\r\n", "crlf")):
        for name in sorted(S.quality_classes(eol)):
            yield "quality_classes/%s/%s" % (tag, name), lambda eol=eol, name=name: S.quality_classes(eol)[name]
        for end in S.STEP_ENDS:
            yield "step_sweep/%s/%s" % (tag, end), lambda eol=eol, end=end: S.step_sweep(eol, end)
    yield "many_reads", S.many_reads
    for name in sorted(S.INNER_CR):
        yield "inner_cr/" + name, lambda name=name: S.INNER_CR[name]


def select(path, sql):
    con = sqlite3.connect(path)
    rows = [list(r) for r in con.execute(sql)]
    con.close()
    return rows


def fasta_answers(path):
    fa = pyfastx.Fasta(path, full_index=True)
    rec = {}
    for k in ("composition", "gc_content", "gc_skew"):
        try:
            rec[k] = getattr(fa, k)
        except RuntimeError:
            rec[k] = None
    rec["type"] = fa.type
    del fa
    rec["comp_digest"] = S.comp_digest(select(path + ".fxi", "SELECT seqid,abc,num FROM comp ORDER BY ID"))
    return rec


def fastq_answers(path):
    fq = pyfastx.Fastq(path, full_index=True)
    rec = {"composition": fq.composition, "gc_content": fq.gc_content, "maxlen": fq.maxlen, "minlen": fq.minlen,
           "maxqual": fq.maxqual, "minqual": fq.minqual, "phred": fq.phred, "encoding_type": fq.encoding_type}
    del fq
    rec["base"] = select(path + ".fxi", "SELECT * FROM base")
    rec["meta"] = select(path + ".fxi", "SELECT * FROM meta")
    return rec


def main():
    tmp = tempfile.mkdtemp(prefix="fxfull")
    out = {"reference": pyfastx.version(debug=True), "fasta": {}, "fastq": {}}
    for kind, inputs, answers in (("fastq", fastq_inputs, fastq_answers), ("fasta", fasta_inputs, fasta_answers)):
        for i, (name, make) in enumerate(inputs()):
            print(kind, name, flush=True)
            data = make()
            assert kind == "fastq" or data.isascii(), name
            path = os.path.join(tmp, "c%d.%s" % (i, "fa" if kind == "fasta" else "fq"))
            with open(path, "wb") as f:
                f.write(data)
            out[kind][name] = answers(path)
            os.remove(path)
            os.remove(path + ".fxi")
    dst = os.path.join(HERE, "full_stats.json.gz")
    with gzip.GzipFile(dst, "wb", mtime=0) as g:
        g.write(json.dumps(out, sort_keys=True, indent=0).encode())
    shutil.rmtree(tmp)
    print("wrote", dst, os.path.getsize(dst), "bytes;", len(out["fasta"]) + len(out["fastq"]), "inputs")


if __name__ == "__main__":
    main()
