#!/usr/bin/env python3
"""Generate tests/golden/edge_layouts.json.gz from the UNMODIFIED reference (oracle/_ref build): what the reference
writes and returns for the byte-level edge patterns of tests/edgelib.py, each as a small file and, for a handful, placed
on the scan's region / window edges.  For every input:

- FASTA: the `seq` rows and `stat` of its .fxi, the `comp` rows of a full index (not for inputs with bytes >= 0x80,
  where the reference indexes a 128-entry array out of bounds), and digests (goldenlib.text_digest) of every record's
  whole `.seq` / `.antisense` and of one slice of it;
- FASTQ: the `read` rows and `stat`, and the `base` / `meta` rows of a full index.

    bash oracle/build_ref.sh && python tests/golden/make_golden_edges.py

tests/test_edge_layouts_cpu.py pins the CPU oracle and the numpy restatements in edgelib to these answers."""
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
import edgelib as E  # noqa: E402
import goldenlib as G  # noqa: E402

# placed inputs compared with the reference besides the small catalogue files
PLACED = ("fasta:crlf_header_cr/small/d0", "fasta:header_start/small/d2", "fasta:name_space_64/small/d1",
          "fasta:crlf_seq_lf/small/d0", "fasta:no_newline_at_end/32768+0/d0", "fasta:header_at_eof_nl/32768-1/d2",
          "fastq:crlf_split_seq/small/d2", "fastq:qual_starts_at/small/d0", "fastq:partial_tail/32768+0/d0")


def inputs():
    """name -> bytes of every input the golden file covers"""
    out = {"small:" + k: E.small_file(p) for k, p in E.CATALOGUE.items()}
    for key in PLACED:
        out["placed:" + key] = E.build(key)[0]
    return out


def select(path, sql):
    con = sqlite3.connect(path)
    con.text_factory = bytes
    rows = [[x.decode("latin-1") if isinstance(x, bytes) else x for x in r] for r in con.execute(sql)]
    con.close()
    return rows


def slice_of(slen):
    return slen // 3, slen - slen // 4


def fasta_answers(path, data):
    fa = pyfastx.Fasta(path)
    rec = {"rows": select(path + ".fxi", "SELECT * FROM seq ORDER BY ID"),
           "stat": select(path + ".fxi", "SELECT * FROM stat")[0][:2], "whole": [], "slice": []}
    for i in range(len(fa)):
        s = fa[i]
        rec["whole"].append([G.text_digest(s.seq), G.text_digest(s.antisense)])
    del fa
    fb = pyfastx.Fasta(path)                 # slices on an object of their own (the reference's cache window)
    for i in range(len(fb)):
        a, b = slice_of(len(fb[i]))
        sub = fb[i][a:b] if b > a else None
        rec["slice"].append(None if sub is None else [G.text_digest(sub.seq), G.text_digest(sub.antisense)])
    del fb
    if not any(x >= 128 for x in data):
        os.remove(path + ".fxi")
        fc = pyfastx.Fasta(path, full_index=True)
        del fc
        rec["comp"] = select(path + ".fxi", "SELECT seqid,abc,num FROM comp ORDER BY ID")
    return rec


def fastq_answers(path):
    fq = pyfastx.Fastq(path, full_index=True)
    del fq
    return {"rows": select(path + ".fxi", "SELECT * FROM read ORDER BY ID"),
            "stat": select(path + ".fxi", "SELECT * FROM stat")[0],
            "base": select(path + ".fxi", "SELECT * FROM base"), "meta": select(path + ".fxi", "SELECT * FROM meta")}


def main():
    tmp = tempfile.mkdtemp(prefix="fxedge")
    out = {"reference": pyfastx.version(debug=True), "cases": {}}
    for i, (name, data) in enumerate(sorted(inputs().items())):
        print("case", name, flush=True)
        fasta = name.split(":")[1] == "fasta"
        path = os.path.join(tmp, "c%d.%s" % (i, "fa" if fasta else "fq"))
        with open(path, "wb") as f:
            f.write(data)
        out["cases"][name] = fasta_answers(path, data) if fasta else fastq_answers(path)
    dst = os.path.join(HERE, "edge_layouts.json.gz")
    with gzip.GzipFile(dst, "wb", mtime=0) as g:
        g.write(json.dumps(out, sort_keys=True).encode())
    shutil.rmtree(tmp)
    print("wrote", dst, os.path.getsize(dst), "bytes;", len(out["cases"]), "cases")


if __name__ == "__main__":
    main()
