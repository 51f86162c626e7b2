"""Expected answers of the search with mismatches, from the CPU oracle's haystacks (searchlib.haystacks for FASTA
queries, readsearchlib.read_haystacks for FASTQ reads): for every start i with i + m <= len(hay), the number of positions
j where hay[i + j] != P[j], for P (plus strand) and for searchlib.revcomp(P) (minus strand).  A hit is a start whose
count is at most k; it is reported as (query, start, minus, mismatches)."""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

import searchlib as S


def window_mismatches(hay, pat):
    """per start i of hay with i + len(pat) <= len(hay): the bytes of hay[i, i + m) that differ from pat"""
    h, p = np.frombuffer(hay, np.uint8), np.frombuffer(pat, np.uint8)
    if h.size < p.size:
        return np.zeros(0, dtype=np.int64)
    return (sliding_window_view(h, p.size) != p).sum(axis=1)


def strand_counts(hays, pat, strands=3):
    """[(plus counts, minus counts)] per haystack (None for a strand not in `strands`): what expected_from_counts needs,
    computed once for several k"""
    rc = S.revcomp(pat)
    return [(window_mismatches(h, pat) if strands & 1 else None, window_mismatches(h, rc) if strands & 2 else None)
            for h in hays]


def expected_from_counts(counts, k, strands=1):
    hits = []
    for q, cs in enumerate(counts):
        for minus in (0, 1):
            if (strands >> minus) & 1:
                c = cs[minus]
                hits += [(q, int(i), minus, int(c[i])) for i in np.flatnonzero(c <= k)]
    return sorted(hits)


def expected_hits(hays, pat, k, strands=1):
    """sorted (query, start, minus, mismatches) of every start within k mismatches; strands: bit 0 plus, bit 1 minus"""
    return expected_from_counts(strand_counts(hays, pat, strands), k, strands)
