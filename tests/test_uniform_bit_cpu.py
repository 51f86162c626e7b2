"""The uniform-lines bit (FASTA row pad[0] & 1) without a GPU: the oracle sets it by the rule of fasta_finalize_kernel,
a plain numpy restatement agrees on random, edge-catalogue and golden inputs, the layouts of tests/uniformlib.py reach
the path each names, and on a record the bit calls uniform the slice formula gives the whole-record strip."""
import numpy as np
import pytest

import edgelib as E
import gatherlib as GL
import gen
import goldenlib as G
import uniformlib as U
from oracle import fxo


def check_bits(data, what):
    rows, _, no_header = fxo.fasta_scan(data)
    if no_header:
        return rows
    want = U.uniform_bits(data)
    bit = rows["pad"][:, 0]
    bad = np.flatnonzero(bit != want)
    assert bad.size == 0, (what, bad[:5], bit[bad[:5]], want[bad[:5]])
    assert (rows["pad"][:, 1:] == 0).all(), what
    assert (rows["norm"][bit == 1] == 1).all(), what                        # uniform implies norm = 1
    assert [int(GL.uniform_of(data, r)) for r in rows] == bit.tolist(), what
    return rows


@pytest.mark.parametrize("seed", range(12))
def test_oracle_bit_matches_numpy_on_random_fasta(seed):
    data = gen.random_fasta(seed, n_records=60 + 20 * seed, no_trailing_newline=(seed % 3 == 0),
                            lead_garbage=(seed % 5 == 1), crlf_prob=0.3 * (seed % 2))
    check_bits(data, seed)


def test_oracle_bit_matches_numpy_on_edge_catalogue_and_golden():
    for key, p in E.CATALOGUE.items():
        if p.kind == "fasta":
            check_bits(E.small_file(p), key)
    for key, (pk, sites, dense) in E.layouts().items():
        if pk.startswith("fasta:") and "8MiB" not in key:
            check_bits(E.build(key)[0], key)
    for case in G.cases("fasta"):
        check_bits(G.case_data(case), case["name"])


def test_last_line_without_newline_counts_its_virtual_newline():
    """a last line of bpl + 1 letters at the end of the file is as long as the others plus one: not uniform; one of
    bpl letters is uniform"""
    for tail, uni in ((b"ACGTA", 0), (b"ACGT", 1), (b"ACG", 1)):
        data = b">a\nACGT\nACGT\n" + tail
        rows = check_bits(data, tail)
        assert int(rows["pad"][0, 0]) == uni, tail


def all_family_layouts():
    return list(U.layouts().values())


def rec_rows(lay):
    rows, _, _ = fxo.fasta_scan(lay.data)
    names = [n.decode() for n in fxo.fasta_names(lay.data, rows)]
    return rows, [names.index(r.name) for r in lay.recs]


@pytest.mark.parametrize("name", sorted(U.layouts()))
def test_layout_bits_and_paths(name):
    """the oracle gives every layout record the bit and norm it was built for, the numpy restatement agrees on the whole
    file, and the record's last newline lies where the path its family names settles it"""
    lay = U.layouts()[name]
    rows, idx = rec_rows(lay)
    check_bits(lay.data, name)
    for r, i, at, path in zip(lay.recs, idx, lay.anchors, lay.paths):
        assert (int(rows["pad"][i, 0]), int(rows["norm"][i])) == (int(r.uniform), int(r.norm)), r.name
        p = int(rows["boff"][i]) + int(rows["blen"][i]) - 1            # the last newline, or the virtual one at n
        assert p == at, r.name
        assert (lay.data[p:p + 1] == b"\n") or (p == len(lay.data) and r.tail), r.name
        assert U.settled_by(lay.data, p) == path, (r.name, U.settled_by(lay.data, p), path)


def test_families_cover_every_variant_and_path():
    seen = set()
    for lay in U.layouts().values():
        for r, path in zip(lay.recs, lay.paths):
            seen.add((path, r.variant, r.tail))
    for path in ("fact", "rows01", "general", "dense", "carry"):
        for v in ("minus1", "plus1", "empty"):
            assert (path, v, False) in seen and (path, v, True) in seen, (path, v)
    assert {("carry", "kib", False), ("carry", "kib", True)} <= seen
    # the carry family: the region before the last line's region with 0 or 1 newlines, > 64 KiB back, and dense
    back = {}
    for fam in ("carry_2k", "carry_64k", "carry_dense"):
        lay = U.layouts()[fam + "_nl"]
        at = lay.anchors[0]
        r = at // U.REGION
        back[fam] = E.region_view(lay.data, (r - 1) * U.REGION)[0]
    assert back["carry_2k"] < 2 and back["carry_64k"] < 2 and back["carry_dense"] > U.SEGCAP
    lay = U.layouts()["carry_64k_nl"]
    assert lay.anchors[0] - lay.data.rfind(b"\n", 0, lay.anchors[0]) > 64 * 1024


@pytest.mark.parametrize("shift,variant", U.block_keys())
def test_block_layouts(shift, variant):
    lay = U.block_layout(shift, variant)
    rows, idx = rec_rows(lay)
    check_bits(lay.data, lay.name)
    r, i, at = lay.recs[0], idx[0], lay.anchors[0]
    assert at == U.BLOCK_BYTES + shift and lay.data[at:at + 1] == b"\n"
    assert int(rows["boff"][i]) + int(rows["blen"][i]) - 1 == at
    assert int(rows["pad"][i, 0]) == int(r.uniform) == (variant == "minus1")
    if shift in (0, 1):            # lines 0 and 1 of the first region of the second prefix block
        nl, facts, k = E.region_view(lay.data, at)
        assert at // U.REGION == 4096 and k in (0, 1) and U.settled_by(lay.data, at) == "rows01"


@pytest.mark.parametrize("world", U.SHARD_WORLDS)
def test_shard_cuts_start_every_record(world):
    data, recs, starts = U.shard_layout()
    check_bits(data, "shard")
    firsts = set()
    for cuts in U.shard_cuts(world):
        assert len(cuts) == world - 1 and cuts == sorted(set(cuts))
        for c in cuts:
            assert data[c:c + 1] == b">"
            firsts.add(c)
    assert firsts == set(starts)
    # the 3000-column records' last newline lies past the second region of their shard
    for r, st in zip(recs, starts):
        if r.name.startswith("w"):
            assert r.anchor >= 2 * U.REGION


def formula_vs_strip(data, rows, i, s, e):
    """(formula-range strip, whole-record strip[s:e]) of each window of row i, packed: fxo.subseq_batch on the row with
    norm forced to 1, and slices of the whole record fxo.subseq strips with the WHOLE flag"""
    r1 = rows.copy()
    r1["norm"] = 1
    rid = np.full(s.size, i, np.int64)
    a, _, _ = fxo.subseq_batch(data, r1, rid, s, e, np.zeros(s.size, np.int32))
    whole = np.frombuffer(fxo.subseq(data, rows[i], 0, int(rows["slen"][i]), fxo.WHOLE), np.uint8)
    b = np.concatenate([whole[x:y] for x, y in zip(s, e)])
    return a, b


def record_windows(row, rec):
    """windows() plus every start within 160 letters of the last two line breaks and of the end, each 7 letters long and
    running to the end"""
    slen = int(row["slen"])
    out = set(U.windows(row, rec))
    bpl = int(row["llen"]) - int(row["elen"])
    starts = set()
    for c in (rec.last_start - bpl, rec.last_start, rec.last_start + bpl, slen):
        starts.update(range(max(0, c - 160), min(slen, c + 160)))
    for x in starts:
        out.add((x, slen))
        out.add((x, min(slen, x + 7)))
    return sorted(out)


def test_formula_equals_strip_exactly_on_uniform_records():
    """the property the kernels rely on: on every record the oracle marks uniform, the formula-range strip equals the
    whole-record strip for every window of the sample; on every record it does not mark uniform, some window differs"""
    lays = all_family_layouts() + [U.block_layout(0, "minus1"), U.block_layout(1, "plus1")]
    n_uniform = n_other = 0
    for lay in lays:
        rows, idx = rec_rows(lay)
        for r, i in zip(lay.recs, idx):
            w = record_windows(rows[i], r)
            s = np.array([x for x, _ in w], np.int64)
            e = np.array([y for _, y in w], np.int64)
            a, b = formula_vs_strip(lay.data, rows, i, s, e)
            if rows["pad"][i, 0]:
                n_uniform += 1
                bad = np.flatnonzero(a != b)
                assert bad.size == 0, (lay.name, r.name, bad[:3])
            else:
                n_other += 1
                assert (a != b).any(), (lay.name, r.name)
    assert n_uniform >= 100 and n_other >= 100
