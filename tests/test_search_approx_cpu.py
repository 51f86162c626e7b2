"""Search with mismatches without a GPU: both entry points fail loudly, their declarations parse from the header, the hit
record carries the mismatch count where the header puts it, and the expectation the GPU tests compare against gives
hand-computed answers."""
import ctypes as C
import gzip
import os
import re

import numpy as np
import pytest

import approxlib as A
import goldenlib as G
import readsearchlib as R
import searchlib as S
from pyfastx_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fxg.h")).read(), flags=re.S)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_search_approx_without_device_is_enodev():
    lib = _cabi.lib()
    out, n = C.c_void_p(), C.c_int64(-1)
    rc = lib.fxg_search_approx_host(None, None, None, 0, None, None, None, 0, 0, b"ACGT", 4, 1, _cabi.SEARCH_PLUS,
                                    C.byref(out), C.byref(n))
    assert rc == _cabi.FXG_ENODEV
    assert b"no CPU fallback" in lib.fxg_last_error()
    rc = lib.fxg_search_reads_approx_host(None, None, None, 0, b"ACGT", 4, 1, _cabi.SEARCH_PLUS, C.byref(out), C.byref(n))
    assert rc == _cabi.FXG_ENODEV
    assert b"no CPU fallback" in lib.fxg_last_error()


@pytest.mark.parametrize("name, arity, rows_type", [("fxg_search_approx_host", 15, "const fxg_fasta_row *"),
                                                    ("fxg_search_reads_approx_host", 10, "const fxg_fastq_row *")])
def test_search_approx_declarations_parse_from_header(name, arity, rows_type):
    m = re.search(r"int\s+%s\s*\(([^;]*)\);" % name, _header())
    assert m, "%s is not declared" % name
    params = [p.strip() for p in m.group(1).split(",")]
    assert len(params) == len(_cabi.SIGNATURES[name][1]) == arity
    assert params[2].startswith(rows_type)
    assert params[arity - 4] == "int32_t max_mismatches" and params[arity - 5] == "int32_t m"
    assert params[arity - 2].startswith("fxg_search_hit **")
    assert name in _cabi.declared_symbols()


def test_hit_record_carries_mismatches_at_byte_20():
    assert _cabi.SEARCH_HIT.itemsize == 24
    assert _cabi.SEARCH_HIT.names == ("query", "start", "minus", "mismatches")
    assert _cabi.SEARCH_HIT.fields["mismatches"][1] == 20
    assert re.search(r"typedef struct fxg_search_hit \{ int64_t query, start; int32_t minus, mismatches; \} fxg_search_hit;",
                     _header())


def test_zero_mismatches_is_the_exact_expectation():
    data = gzip.open(os.path.join(G.GOLD, "data", "test.fa.gz")).read()
    _, hays = S.whole_records(data)
    for pat in (b"GCTTCAATACA", b"ACGT", b"GAATTC", b"T", b"CCGG"):
        for mask in (1, 2, 3):
            assert A.expected_hits(hays, pat, 0, mask) == [h + (0,) for h in S.expected_hits(hays, pat, mask)], pat


def test_expectation_on_hand_made_reads():
    data = (b"@r0\nAACCGG\n+\nIIIIII\n"
            b"@r1\nTTTACG\n+\nIIIIII\n"
            b"@r2\r\nNNAcg\xe9\r\n+\r\nIIIII\r\n")
    rows, hays = R.read_haystacks(data)
    assert hays == [b"AACCGG", b"TTTACG", b"NNAcg\xe9"]
    # CCGT: AACC 4, ACCG 3, CCGG 1; its reverse complement ACGG: AACC 3, ACCG 1, CCGG 1; against TTTACG and NNAcg\xe9
    # every window differs in all four bytes
    assert A.expected_hits(hays, b"CCGT", 1, 3) == [(0, 1, 1, 1), (0, 2, 0, 1), (0, 2, 1, 1)]
    assert A.expected_hits(hays, b"CCGT", 3, 1) == [(0, 1, 0, 3), (0, 2, 0, 1)]
    # ACGT would be ACG + one missing byte at the end of r1: a window never runs past its read's end
    assert A.expected_hits(hays, b"ACGT", 1, 1) == []
    # ACGT: AACC 3, ACCG 2, CCGG 2; TTTA, TTAC, TACG 4 each; NNAc 4, NAcg 4, Acg\xe9 3
    assert A.expected_hits(hays, b"ACGT", 3, 1) == [(0, 0, 0, 3), (0, 1, 0, 2), (0, 2, 0, 2), (2, 2, 0, 3)]
    assert all(s + 4 <= len(hays[q]) for q, s, _, _ in A.expected_hits(hays, b"ACGT", 3, 3))
    # byte for byte and case-sensitive: N against A and c against C are mismatches
    assert A.expected_hits(hays, b"NAAcg", 1, 1) == [(2, 0, 0, 1)]
    assert A.expected_hits(hays, b"NNACG", 1, 1) == []
    assert A.expected_hits(hays, b"NNACG", 2, 1) == [(1, 1, 0, 2), (2, 0, 0, 2)]       # TTACG and NNAcg
    # an A-run: a pattern with one A and k = m - 1 hits at every start
    assert A.expected_hits([b"A" * 9], b"CAG", 2, 1) == [(0, i, 0, 2) for i in range(7)]
    assert np.array_equal(A.window_mismatches(b"AC", b"ACG"), np.zeros(0, np.int64))
