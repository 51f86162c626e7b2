"""Expected pattern-search answers in FASTQ reads from the CPU oracle: the haystack of a read is its sequence bytes as
the oracle fetches them (Read.seq: the raw rlen bytes at soff), and hits are found as in searchlib."""
from oracle import fxo


def read_haystacks(data):
    """oracle rows of the complete FASTQ reads and the haystack of each: its sequence bytes (Read.seq)"""
    rows, _, _ = fxo.fastq_scan(data)
    return rows, [fxo.read_fetch(data, r)[0] for r in rows]
