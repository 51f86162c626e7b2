"""N>1 host logic (pyfastx_b200/shard.py) on CPU: world_size-2 and -3 gloo process groups.  Every rank cuts the
file at split points found on the data, scans its own byte range (a pure-Python stand-in plays the two device
phases fxg_scan_begin / fxg_scan_finish; the GPU kernels themselves are covered by tests/test_gpu_parity.py and
by the 2-GPU run of tools/check_sharded.py), ONE all-gather of the 128-byte shard infos, boundary-row merge from
the gathered edge lines, rows to rank 0 -- and the merged result must equal the whole-file oracle."""
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _lines(data):
    """[(start, length without '\\n')] incl. an unterminated last line (kseq semantics)"""
    out, pos = [], 0
    for ln in data.split(b"\n"):
        out.append((pos, len(ln)))
        pos += len(ln) + 1
    if out and data.endswith(b"\n"):
        out.pop()
    if not data:
        out = []
    return out


def py_begin(data, base_offset, mode):
    """stand-in for fxg_scan_begin: the shard's fxg_shard_info"""
    from pyfastx_b200._cabi import SHARD_INFO
    ls = _lines(data)
    info = np.zeros(1, dtype=SHARD_INFO)[0]
    info["n_lines"] = len(ls)
    info["bytes"] = len(data)
    info["base_offset"] = base_offset
    info["n_rows"] = sum(1 for s, l in ls if data[s:s + 1] == b">") if mode == 0 else 0
    info["edge_n"] = min(3, len(ls))
    for j, (s, l) in enumerate(ls[:3]):
        info["edge_off"][j] = base_offset + s
        info["edge_len"][j] = l - (1 if l > 0 and data[s + l - 1:s + l] == b"\r" else 0)
    return info


def py_finish_fastq(data, base_offset, infos, rank):
    """stand-in for fxg_scan_finish (FASTQ): rows of the reads whose name line lies in this shard"""
    from pyfastx_b200 import shard
    from pyfastx_b200._cabi import FASTQ_ROW
    first, first_read, owned, n_reads = shard.fastq_layout(infos["n_lines"])
    F, n = int(first[rank]), int(infos["n_lines"][rank])
    ls = _lines(data)

    def line(g):                       # (global offset, rlen-style length) of global line g
        if F <= g < F + n:
            s, l = ls[g - F]
            return base_offset + s, l - (1 if l > 0 and data[s + l - 1:s + l] == b"\r" else 0)
        for p in range(rank + 1, len(infos)):
            Fp, np_ = int(first[p]), int(infos["n_lines"][p])
            if Fp <= g < Fp + np_:
                j = g - Fp
                assert j < int(infos["edge_n"][p])
                return int(infos["edge_off"][p][j]), int(infos["edge_len"][p][j])
        raise AssertionError("line %d not found" % g)

    rows = np.zeros(int(owned[rank]), dtype=FASTQ_ROW)
    size = 0
    for g in range(F, F + n):
        if g % 4 == 1:
            size += line(g)[1]
    for i in range(len(rows)):
        R = int(first_read[rank]) + i
        s, l = ls[4 * R - F]
        name = data[s + 1:s + l].rstrip(b"\r") if l > 0 else b""
        if b"\x00" in name.split(b" ")[0]:
            k = len(name)
        else:
            k = name.find(b" ")
        rows[i]["dlen"] = l
        rows[i]["nlen"] = len(name) if k < 0 else k
        rows[i]["soff"], rows[i]["rlen"] = line(4 * R + 1)
        rows[i]["qoff"] = line(4 * R + 3)[0]
    return rows, size


def _all_gather_infos(info):
    from pyfastx_b200._cabi import SHARD_INFO
    t = torch.from_numpy(np.frombuffer(info.tobytes(), dtype=np.uint8).copy())
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return np.frombuffer(b"".join(o.numpy().tobytes() for o in out), dtype=SHARD_INFO).copy()


def _worker(rank, world, port, fa, fq, fq_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from oracle import fxo
    from pyfastx_b200 import shard
    # ---- FASTA: shards start at header lines found on the data ------------------------------------------
    pts = shard.fasta_split_points(fa, world)
    a, b = pts[rank], pts[rank + 1]
    infos = _all_gather_infos(py_begin(fa[a:b], a, 0))
    if b > a:
        rows, total, _ = fxo.fasta_scan(fa[a:b])
        rows["boff"] += a
    else:
        rows, total = np.zeros(0, dtype=fxo.FASTA_ROW), 0
    assert int(infos["n_rows"][rank]) == len(rows)
    base, n_total = shard.fasta_layout(infos["n_rows"])
    fa_parts = shard.gather_objects((rows, total))
    # the raw-byte gather used by build_index_sharded must deliver the same arrays (structured rows, an empty array,
    # int64 offsets) as the pickling one
    raw_parts = shard.gather_arrays((rows, np.zeros(0 if rank else 3, dtype=np.uint8), np.arange(rank + 2, dtype=np.int64)))
    if rank == 0:
        assert len(raw_parts) == world
        for r in range(world):
            assert raw_parts[r][0].dtype == rows.dtype and np.array_equal(raw_parts[r][0], fa_parts[r][0])
            assert raw_parts[r][1].size == (0 if r else 3)
            assert np.array_equal(raw_parts[r][2], np.arange(r + 2, dtype=np.int64))
    else:
        assert raw_parts is None
    # ---- FASTQ: shards start at line starts; global line phase from the gathered line counts -----------------
    lp = shard.line_split_points(fq, world)
    assert lp == shard.split_points_path(fq_path, world, False)          # pread search == in-memory search
    la, lb = lp[rank], lp[rank + 1]
    qinfos = _all_gather_infos(py_begin(fq[la:lb], la, 1))
    qrows, qsize = py_finish_fastq(fq[la:lb], la, qinfos, rank)
    fq_parts = shard.gather_objects((qrows, qsize))
    if rank == 0:
        q.put((n_total, [int(x) for x in base], fa_parts, fq_parts, int(qinfos["n_lines"].sum())))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_host_logic_gloo(world):
    import gen
    from oracle import fxo
    fa = gen.random_fasta(77, n_records=120, crlf_prob=0.0)
    fq = gen.random_fastq(78, n_reads=301, partial_tail=1)
    with tempfile.NamedTemporaryFile(suffix=".fq", delete=False) as tf:
        tf.write(fq)
        fq_path = tf.name
    try:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_worker, args=(r, world, port, fa, fq, fq_path, q)) for r in range(world)]
        for p in procs:
            p.start()
        n_total, base, fa_parts, fq_parts, n_lines = q.get(timeout=120)
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        os.unlink(fq_path)
    exp, exp_total, _ = fxo.fasta_scan(fa)
    got = np.concatenate([p[0] for p in fa_parts])
    assert n_total == len(exp) and sum(p[1] for p in fa_parts) == exp_total
    assert base == np.concatenate([[0], np.cumsum([len(p[0]) for p in fa_parts])[:-1]]).tolist()
    for f in ("boff", "blen", "slen", "llen", "dlen", "nlen", "elen", "norm", "pad"):
        assert np.array_equal(got[f], exp[f]), f
    qexp, qsize, qlines = fxo.fastq_scan(fq)
    qgot = np.concatenate([p[0] for p in fq_parts])
    assert n_lines == qlines and sum(p[1] for p in fq_parts) == qsize and len(qgot) == len(qexp)
    for f in ("soff", "qoff", "rlen", "dlen", "nlen"):
        assert np.array_equal(qgot[f], qexp[f]), f


def test_split_points_are_on_the_data():
    from pyfastx_b200 import shard
    fa = b">a\nACGT\nAC\n>b x\nGG\n>c\nTTTT\nTT\n"
    for world in (1, 2, 3, 5, 9):
        pts = shard.fasta_split_points(fa, world)
        assert pts[0] == 0 and pts[-1] == len(fa) and pts == sorted(pts)
        for p in pts[1:-1]:
            assert p == len(fa) or (fa[p:p + 1] == b">" and fa[p - 1:p] == b"\n")
        lp = shard.line_split_points(fa, world)
        for p in lp[1:-1]:
            assert p == len(fa) or fa[p - 1:p] == b"\n"
    first, first_read, owned, n_reads = shard.fastq_layout([5, 1, 0, 2, 9])
    assert first.tolist() == [0, 5, 6, 6, 8] and n_reads == 4
    assert first_read.tolist() == [0, 2, 2, 2, 2] and owned.tolist() == [2, 0, 0, 0, 2]
