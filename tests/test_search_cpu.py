"""Pattern search (K8) without a GPU: the entry point fails loudly, its limits parse from the header, and the
oracle-haystack expectation the GPU tests compare against reproduces the reference's documented answer."""
import ctypes as C
import gzip
import os
import re

import numpy as np
import pytest

import goldenlib as G
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
def test_search_without_device_is_enodev():
    lib = _cabi.lib()
    out, n = C.c_void_p(), C.c_int64(-1)
    rc = lib.fxg_search_host(None, None, None, 0, None, None, None, 0, 0, b"ACGT", 4, _cabi.SEARCH_PLUS,
                             _cabi.SEARCH_ALL, C.byref(out), C.byref(n))
    assert rc == _cabi.FXG_ENODEV
    assert b"no CPU fallback" in lib.fxg_last_error()


def test_search_limits_parse_from_header():
    text = open(os.path.join(ROOT, "include", "fxg.h")).read()
    piece = int(re.search(r"#define\s+FXG_SEARCH_PIECE\s+(\d+)", text).group(1))
    cap = int(re.search(r"#define\s+FXG_SEARCH_MAX_PATTERN\s+(\d+)", text).group(1))
    assert (piece, cap) == (_cabi.SEARCH_PIECE, _cabi.SEARCH_MAX_PATTERN)
    assert piece % 128 == 0 and piece >= cap + 512
    assert _cabi.SEARCH_HIT.itemsize == 24 and "} fxg_search_hit;" in text
    for needle in ("src/sequence.c:519-560", "src/util.c:769-783"):
        assert needle in text


def test_expectation_reproduces_reference_answer():
    """README of the reference: fa[0].search('GCTTCAATACA') == 262 on tests/data/test.fa.gz"""
    data = gzip.open(os.path.join(G.GOLD, "data", "test.fa.gz")).read()
    rows, hays = S.whole_records(data)
    assert len(rows) == 211
    assert S.first_position(hays[0], b"GCTTCAATACA", False) == 262
    hits = S.expected_hits(hays[:1], b"GCTTCAATACA", 3)
    assert (0, 261, 0) in hits
    # overlapping occurrences all count; a palindrome is reported once per strand
    assert S.occurrences(b"AAAAAAA", b"AAAA") == [0, 1, 2, 3]
    assert S.expected_hits([b"xxGAATTCxx"], b"GAATTC", 3) == [(0, 2, 0), (0, 2, 1)]
    assert S.revcomp(b"ACGTNacgtnRYKMBVDHU\xe9") == b"\xe9ADHBVKMRYnacgtNACGT"
