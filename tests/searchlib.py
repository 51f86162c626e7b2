"""Expected pattern-search answers from the CPU oracle: the haystack of a query is what the oracle extracts for it
(fxo.subseq_batch), and a hit is every overlapping occurrence of the pattern (plus strand) or of its reverse
complement under the extraction complement table (minus strand), reported by its 0-based forward start."""
import numpy as np

from oracle import fxo


def revcomp(pat):
    lut = fxo.complement_lut()
    return bytes(lut[np.frombuffer(pat, dtype=np.uint8)][::-1]) if pat else b""


def occurrences(hay, pat):
    """0-based starts of every (overlapping) occurrence of pat in hay"""
    out, k = [], hay.find(pat)
    while k >= 0:
        out.append(k)
        k = hay.find(pat, k + 1)
    return out


def haystacks(data, rows, rid, s, e, upper=False):
    rid = np.asarray(rid, dtype=np.int64)
    flags = np.full(rid.size, fxo.UPPER if upper else 0, dtype=np.int32)
    out, off, _ = fxo.subseq_batch(data, rows, rid, s, e, flags)
    buf = out.tobytes()
    return [buf[off[i]:off[i + 1]] for i in range(rid.size)]


def expected_hits(hays, pat, strands=1):
    """sorted (query, start, minus) of every hit; strands: bit 0 plus, bit 1 minus"""
    rc = revcomp(pat)
    hits = []
    for q, h in enumerate(hays):
        if strands & 1:
            hits += [(q, k, 0) for k in occurrences(h, pat)]
        if strands & 2:
            hits += [(q, k, 1) for k in occurrences(h, rc)]
    return sorted(hits)


def first_hits(hits):
    """the first hit of each (query, strand) of a sorted hit list, in (query, start, minus) order"""
    first = {}
    for q, k, mi in hits:
        first.setdefault((q, mi), k)
    return sorted((q, k, mi) for (q, mi), k in first.items())


def first_position(hay, pat, minus):
    """what Sequence.search answers: the 1-based start of the first hit, or None"""
    k = hay.find(revcomp(pat) if minus else pat)
    return k + 1 if k >= 0 else None


def whole_records(data, upper=False):
    """oracle rows and the haystack of every whole record"""
    rows, _, _ = fxo.fasta_scan(data)
    n = len(rows)
    return rows, haystacks(data, rows, np.arange(n), np.zeros(n, np.int64), rows["slen"], upper)
