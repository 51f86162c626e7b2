"""Pattern search in FASTQ reads without a GPU: the entry point fails loudly, its declaration parses from the header, and
the oracle-read expectation the GPU tests compare against gives known answers on hand-made reads."""
import ctypes as C
import os
import re

import pytest

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


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_search_reads_without_device_is_enodev():
    lib = _cabi.lib()
    out, n = C.c_void_p(), C.c_int64(-1)
    rc = lib.fxg_search_reads_host(None, None, None, 0, b"ACGT", 4, _cabi.SEARCH_PLUS, C.byref(out), C.byref(n))
    assert rc == _cabi.FXG_ENODEV
    assert b"no CPU fallback" in lib.fxg_last_error()


def test_search_reads_declaration_parses_from_header():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fxg.h")).read(), flags=re.S)
    m = re.search(r"int\s+fxg_search_reads_host\s*\(([^;]*)\);", text)
    assert m, "fxg_search_reads_host is not declared"
    params = [p.strip() for p in m.group(1).split(",")]
    assert len(params) == len(_cabi.SIGNATURES["fxg_search_reads_host"][1]) == 9
    assert params[2].startswith("const fxg_fastq_row *") and params[4].startswith("const uint8_t *")
    assert params[7].startswith("fxg_search_hit **")
    assert "fxg_search_reads_host" in _cabi.declared_symbols()


def test_read_expectation_on_hand_made_reads():
    # sequence, '+' line and quality made of A/C/G/T; names too
    data = (b"@ACGT\nAACCGG\n+\nTTGGAC\n"                 # read 0
            b"@GGTT\r\nAC GT\tA\r\n+\r\nACGTAC\r\n"        # read 1: CRLF, a space and a tab inside the sequence
            b"@CC\nacgNN\xe9\n+\nIIIIII\n"                 # read 2: lower case, N, a byte >= 0x80
            b"@TAIL\nGAATTC\n+\n")                         # a partial record: not a read
    rows, hays = R.read_haystacks(data)
    assert len(rows) == 3
    assert hays == [b"AACCGG", b"AC GT\tA", b"acgNN\xe9"]
    # across the sequence line's end into '\n+\n' or '\r', across the quality line into the next name, across two
    # reads' sequences (GG + AC), a quality line, the partial record
    for pat in (b"GG\n+\nTT", b"GG\n", b"A\r\n+", b"AC\n@GG", b"GGAC", b"TTGGAC", b"GAATTC"):
        assert S.expected_hits(hays, pat, 3) == [], pat
    assert S.expected_hits(hays, b"AC GT", 1) == [(1, 0, 0)]
    assert S.expected_hits(hays, b"ACGT", 3) == []
    assert S.expected_hits(hays, b"CCGG", 3) == [(0, 2, 0), (0, 2, 1)]          # a palindrome: once per strand
    assert S.expected_hits(hays, b"GGTT", 3) == [(0, 0, 1)]                      # its reverse complement AACC
    assert S.expected_hits(hays, b"acg", 3) == [(2, 0, 0)]
    assert S.expected_hits(hays, b"N\xe9", 3) == [(2, 4, 0)]
    assert S.expected_hits([b"A" * 7], b"AAAA", 3) == [(0, k, 0) for k in range(4)]
