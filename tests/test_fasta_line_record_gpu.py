"""FASTA scan edges of the per-region line record: mark settles the lines k >= 2 of a 2 KiB region into at most three
line facts (with the name cut searched over the first 64 header bytes); regions with more newlines or facts take the
general path, lines 0 and 1 of every region are resolved from the region before it.  Every input here is compared
row for row with the oracle; test_fasta_line_record_cpu.py checks that the inputs reach the edges they are named for."""
import numpy as np
import pytest

from oracle import fxo
from pyfastx_b200 import engine, shard

from test_gpu_parity import assert_rows_equal, check_fasta_vs_oracle, emulate_sharded
from test_fasta_line_record_cpu import CASES, rand_fasta

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    return engine.get_engine(0)


@pytest.mark.parametrize("full_name", [False, True])
@pytest.mark.parametrize("case", sorted(CASES))
def test_line_record_vs_oracle(eng, case, full_name):
    for seed in range(3):
        data = rand_fasta(seed * 7 + 1, **CASES[case])
        check_fasta_vs_oracle(eng, data, nq=200, seed=seed, full_name=full_name)


def shard_info_expected(data, base):
    """fxg_shard_info fields of one shard, computed on the host"""
    a = np.frombuffer(data, np.uint8)
    nl = np.nonzero(a == 10)[0].tolist()
    virt = a.size > 0 and a[-1] != 10
    if virt:
        nl.append(a.size)
    offs, lens, start = [], [], 0
    for p in nl[:3]:
        cr = p > start and p - 1 < a.size and a[p - 1] == 13
        offs.append(base + start)
        lens.append(p - start - (1 if cr else 0))
        start = p + 1
    return len(nl), a.size + (1 if virt else 0), offs, lens


@pytest.mark.parametrize("case", ["facts_edges", "crlf", "long_lines", "short"])
def test_sharded_line_record(eng, case):
    data = rand_fasta(5, **CASES[case])
    exp_rows, exp_total, _ = fxo.fasta_scan(data)
    # cuts at header lines: every shard is a FASTA file of its own
    for world in (2, 3, 5):
        pts = shard.fasta_split_points(data, world)
        res = emulate_sharded(eng, data, pts, 0)
        assert_rows_equal(np.concatenate([r[0] for r in res]), exp_rows)
        assert sum(r[1]["total_len"] for r in res) == exp_total
    # cuts at any line: the shard infos
    for world in (3, 7):
        pts = shard.line_split_points(data, world)
        res = emulate_sharded(eng, data, pts, 0)
        infos = res[0][2]
        for r in range(world):
            n_lines, end, offs, lens = shard_info_expected(data[pts[r]:pts[r + 1]], pts[r])
            info = infos[r]
            assert int(info["n_lines"]) == n_lines and int(info["end_position"]) == end
            assert int(info["edge_n"]) == len(offs)
            assert info["edge_off"][:len(offs)].tolist() == offs and info["edge_len"][:len(lens)].tolist() == lens
