"""Inputs for the FASTA line-record tests (tests/test_fasta_line_record_gpu.py), and the check, on the CPU, that they
reach the edges of the per-region line record: regions with exactly LF_MAX and LF_MAX + 1 line facts, header lines at
k = 0, 1, 2 of a region, header facts longer than the 64 bytes mark searches for the name cut, and regions without a
newline."""
import numpy as np

REGION = 2048
LF_MAX = 3



def region_stats(data):
    """per region with a newline: (newlines, line facts k >= 2, header lines at k = 0 / 1 / 2, longest header fact),
    by the rule mark applies (a virtual newline at n when the file does not end in one)"""
    a = np.frombuffer(data, np.uint8)
    n = a.size
    nl = np.nonzero(a == 10)[0].tolist()
    if n and a[-1] != 10:
        nl.append(n)
    hdr = lambda e: e + 1 < n and a[e + 1] == ord(">")
    is_header_line = {e: (hdr(nl[g - 1]) if g else (n > 0 and a[0] == ord(">"))) for g, e in enumerate(nl)}
    by_reg = {}
    for e in nl:
        by_reg.setdefault(e // REGION, []).append(e)
    out = []
    for r, ent in by_reg.items():
        facts, longest = 0, 0
        hk = set()
        for k in range(len(ent)):
            if is_header_line[ent[k]] and k <= 2:
                hk.add(k)
            if k < 2:
                continue
            p, p1, p2 = ent[k], ent[k - 1], ent[k - 2]
            if hdr(p1) or hdr(p2) or p - p1 != p1 - p2:
                facts += 1
                if hdr(p1):
                    longest = max(longest, p - p1 - 2)
        out.append((len(ent), facts, hk, longest))
    return out


def rand_header(rng, i):
    """names of 1..300 bytes, cut by ' ', by '\\t' or not at all"""
    ln = int(rng.choice([1, 5, 30, 31, 32, 33, 63, 64, 65, 66, 100, 300]))
    name = ("r%d_" % i + "x" * ln)[:max(ln, 1)]
    kind = rng.integers(0, 3)
    if kind == 0:
        return ">" + name
    sep = " " if kind == 1 else "\t"
    return ">" + name + sep + "desc%d" % rng.integers(0, 1000)


def rand_fasta(seed, n_records, widths=(60, 80), irregular=0.0, crlf=False, lead=False, trailing_newline=True,
               short=(1, 400), gap_prob=0.0):
    rng = np.random.default_rng(seed)
    eol = "\r\n" if crlf else "\n"
    parts = []
    if lead:
        parts.append("ACGT" * 5 + eol + "AC" + eol)             # lines before the first header: slot 0, lead_llen
    for i in range(n_records):
        parts.append(rand_header(rng, i) + eol)
        if rng.random() < gap_prob:                            # one line longer than a region: regions without a newline
            parts.append("A" * int(rng.integers(2100, 5000)) + eol)
            continue
        L = int(rng.integers(short[0], short[1] + 1))
        w = int(rng.choice(widths))
        s = "".join(rng.choice(list("ACGTN"), size=L))
        pos = 0
        while pos < L:
            ww = w if rng.random() >= irregular else int(rng.integers(1, 2 * w))
            parts.append(s[pos:pos + ww] + eol)
            pos += ww
    data = "".join(parts).encode()
    if not trailing_newline:
        data = data[:-len(eol)]
    return data


CASES = {
    # long records at 80 columns with a few short ones: regions with 0..LF_MAX + 2 facts
    "facts_edges": dict(n_records=400, short=(30, 3000), widths=(80,)),
    # irregular line lengths: length-change facts, many regions over LF_MAX
    "irregular": dict(n_records=300, short=(50, 2500), widths=(70, 80), irregular=0.15),
    # short records: most regions general
    "short": dict(n_records=600, short=(1, 300), widths=(60,)),
    "crlf": dict(n_records=300, short=(30, 3000), widths=(80,), crlf=True),
    "lead_no_trailing_nl": dict(n_records=200, short=(30, 3000), widths=(80,), lead=True, trailing_newline=False),
    # lines longer than a region: the two newlines before a region come from further back
    "long_lines": dict(n_records=200, short=(30, 2000), widths=(80,), gap_prob=0.3),
}


def test_inputs_reach_the_record_edges():
    """the inputs above contain regions with exactly LF_MAX and LF_MAX + 1 facts, header lines at k = 0, 1, 2 of a
    region, header facts longer than the 64 bytes mark searches, and regions without a newline"""
    stats, no_nl = [], 0
    for case, kw in CASES.items():
        for seed in range(3):
            data = rand_fasta(seed * 7 + 1, **kw)
            st = region_stats(data)
            stats += st
            no_nl += (len(data) + REGION - 1) // REGION - len(st)
    small = [s for s in stats if s[0] <= 32]
    assert any(s[1] == LF_MAX for s in small) and any(s[1] == LF_MAX + 1 for s in small)
    for k in (0, 1, 2):
        assert any(k in s[2] for s in stats), k
    assert any(s[3] > 64 and s[1] <= LF_MAX for s in small)
    assert any(32 <= s[3] <= 64 and s[1] <= LF_MAX for s in small)
    assert no_nl > 0
