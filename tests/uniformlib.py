"""Layouts aimed at the FASTA scan's uniform-lines bit (row pad[0] & 1) and at each path that settles it.

The scan keeps, per record, the number of line-length changes D, the line index of the last change and the sum of the
changes S; fasta_finalize_kernel marks a record uniform when D = 0, or when D = 1 and that one change is a SHORTER last
line.  Which code raises the event of a line depends on where its newline falls (tests/edgelib.py, region_view):

- 'fact':    line k >= 2 of a region mark settles (at most 32 newlines, at most 3 line facts): a line fact;
- 'rows01':  line 0 or 1 of such a region, the two newlines before it taken from the previous region's record
             (fasta_rows_kernel's do_line);
- 'carry':   the same lines when the previous region holds fewer than 2 or more than 128 newlines (carry_walk);
- 'general': a region of 33..128 newlines or more than 3 facts (full_region, region_batches);
- 'dense':   a region of more than 128 newlines (full_region, dense_region).

Each layout record has one length change, at its last line (change -1, +1, an empty last line, or several KiB longer),
with LF, CRLF, or a LF last line in a CRLF record; it ends the file with or without a final newline.  Controls: no
change, a change that is not at the last line (norm = 0), and two changes that cancel (norm = 1, not uniform).  A
family places every variant's last newline so that one path settles it; 'block' puts it next to an 8 MiB prefix-block
edge, and shard_layout makes the records the first of a shard.  test_uniform_bit_cpu.py checks on the bytes that each
layout reaches its path."""
import functools

import numpy as np

import edgelib as E

REGION, SEGCAP, BLOCK_BYTES = E.REGION, E.SEGCAP, E.BLOCK_BYTES
KIB = 3000                                   # the "several KiB longer" last line
PATTERN = b"GATTACAGGTCCATTGACCGTATC"        # planted across and inside every record's last line
EOLS = {"lf": (b"\n", b"\n"), "crlf": (b"\r\n", b"\r\n"), "crlf_lf": (b"\r\n", b"\n")}   # (lines, last line)
CHANGES = ("minus1", "plus1", "empty", "kib")
CONTROLS = ("zero", "shift", "cancel")

# family -> (line width, sequence lines, where the last newline goes: offset from a region edge given L_n = len + 1 of
# the last line, the path that settles it)
FAMILIES = {
    "fact":          (80, 60, lambda Ln: 1000, "fact"),
    "rows01_k0":     (80, 60, lambda Ln: 0, "rows01"),
    "rows01_k1":     (80, 60, lambda Ln: 5 + Ln, "rows01"),         # line n - 1 ends at edge + 5
    "carry_2k":      (3000, 4, lambda Ln: 0, "carry"),
    "carry_64k":     (70000, 4, lambda Ln: 0, "carry"),
    "carry_dense":   (6, 800, lambda Ln: 3, "carry"),               # the region before holds ~290 newlines
    "general_lines": (20, 240, lambda Ln: 1000, "general"),
    "general_facts": (80, 4, lambda Ln: 1500, "general"),           # a whole record in one region: 5 facts
    "dense":         (6, 800, lambda Ln: 1500, "dense"),
}
BLOCK_SHIFTS = (-2048, -2047, -1, 0, 1, 2047, 2048)


class Rec:
    """one layout record: bytes, the anchor (index of its last newline, or len(data) for the virtual one), and what
    the scan must give it"""

    def __init__(self, name, data, anchor, uniform, norm, last_start, slen, Ln, tail):
        self.name, self.data, self.anchor = name, data, anchor
        self.uniform, self.norm, self.last_start, self.slen, self.Ln, self.tail = uniform, norm, last_start, slen, Ln, tail

    def pattern(self):
        return E.Pattern(self.name, "fasta", self.data[:self.anchor], self.data[self.anchor:], tail=self.tail)


def _letters(rng, n):
    """A/C/G/T with some soft-masked (lower-case) letters and a few N"""
    a = np.frombuffer(b"ACGTACGTACGTacgtN", np.uint8)[rng.integers(0, 17, size=n)]
    return a


def record(name, width, nlines, eol, variant, final_newline=True, seed=0):
    """-> Rec.  variant: a CHANGES or CONTROLS name; the last line of a change variant is L_1 + change long (len + 1)"""
    rng = np.random.default_rng(seed)
    line_eol, last_eol = EOLS[eol]
    L1 = width + len(line_eol)
    widths = [width] * nlines
    eols = [line_eol] * (nlines - 1) + [last_eol]
    if variant == "minus1":
        widths[-1] = L1 - 1 - len(last_eol)
    elif variant == "plus1":
        widths[-1] = L1 + 1 - len(last_eol)
    elif variant == "empty":
        widths[-1] = 0
    elif variant == "kib":
        widths[-1] = L1 + KIB - len(last_eol)
    elif variant == "zero":
        widths[-1] = L1 - len(last_eol)
    elif variant == "shift":                  # one change, three lines before the end: 2-letter lines from there on
        widths[-3:] = [2, 2, 2]
    elif variant == "cancel":                 # +1 then back: D = 2, S = 0
        widths[-2] = width + 1
    seq = _letters(rng, sum(widths))
    ends = np.cumsum(widths)
    slen = int(ends[-1])
    last_start = slen - widths[-1]
    # inside / at the end / across the last break; one letter before the end: a record that ends the file in a LF line
    # after CRLF lines has one letter more than its slen counts
    for at in (last_start + width + 1, slen - len(PATTERN) - 1, last_start - len(PATTERN) // 2):
        if 0 <= at and at + len(PATTERN) <= slen:
            seq[at:at + len(PATTERN)] = np.frombuffer(PATTERN, np.uint8)
    body = b"".join(bytes(seq[b - w:b]) + e for w, b, e in zip(widths, ends, eols))
    head = b">" + name.encode() + b" " + variant.encode() + line_eol
    data = head + body
    Ln = widths[-1] + len(last_eol)
    if not final_newline:
        data = data[:-1]                      # the virtual newline at the end of the file keeps L_n
        anchor = len(data)
    else:
        anchor = len(data) - 1
    lens = [w + len(e) for w, e in zip(widths, eols)]
    uniform = all(x == lens[0] for x in lens[:-1]) and lens[-1] <= lens[0]
    norm = sum(x != lens[0] for x in lens) <= 1
    rec = Rec(name, data, anchor, uniform, norm, last_start, slen, Ln, not final_newline)
    rec.variant, rec.eol = variant, eol
    return rec


def variants(final_newline=True):
    """(variant, eol) pairs of one family: every change with every line ending, and the controls (LF); without a final
    newline an empty LF last line would not be a line, so those two are left out"""
    out = [(c, e) for c in CHANGES for e in EOLS]
    if final_newline:
        out += [(c, "lf") for c in CONTROLS]
    else:
        out = [(c, e) for c, e in out if not (c == "empty" and EOLS[e][1] == b"\n")]
    return out


# the controls whose own lines move the last newline to another path than the family's
PATH_EXCEPTIONS = {
    ("fact", "cancel"): "general",        # two changes, the next header and its first line: 4 facts
    ("rows01_k1", "shift"): "fact",       # the 3-byte lines before it put the last newline at k = 2
    ("carry_2k", "shift"): "rows01",      # ... and 2 newlines into the region before
    ("carry_64k", "shift"): "rows01",
}


def path_of(variant, family):
    """the path that settles a family's last line.  A last line several KiB long is placed at a region edge: its
    region holds no newline before it and the one before none, so carry_walk finds the two before it."""
    if variant == "kib":
        return "carry"
    return PATH_EXCEPTIONS.get((family, variant), FAMILIES[family][3])


def place_records(recs, at, start=0):
    """file bytes: filler records (edgelib's), then every Rec of recs with its anchor at at(i, rec), each after a run of
    filler; the last one may end the file (rec.tail).  -> (data, anchors)"""
    b = E._Builder("fasta", b"\n", 0)
    if start:
        out, b.rec, b.left = E._prefix("fasta", b"\n", start)
        b.out = bytearray(out)
    anchors = []
    for i, r in enumerate(recs):
        target = at(i, r, len(b.out))
        b.adjust_to(target - r.anchor)
        b.put_pattern(r.pattern())
        anchors.append(target)
        if not r.tail:          # one long filler record after it: its header and first line are the only facts there
            b.out += b">after%d x\n" % i + b"".join((E.S * 4)[k % 60:][:80] + b"\n" for k in range(30))
    if not recs[-1].tail:
        b.fill_to(len(b.out) + 3000)
        while b.left:
            b.push(b.next_item())
    return bytes(b.out), anchors


def _next_edge(pos, rec, off):
    """the first region edge past pos that leaves room for rec's bytes before its anchor, plus off"""
    need = pos + rec.anchor + 3 * REGION
    return (need + REGION - 1) // REGION * REGION + off


class Layout:
    """one file of layout records.  recs[i] is the record whose header follows the names; paths[i] the path its last
    line must take"""

    def __init__(self, name, data, recs, anchors, paths, family):
        self.name, self.data, self.recs, self.anchors, self.paths, self.family = name, data, recs, anchors, paths, family


def family_layouts(family):
    """the family's files: one with every final-newline variant, and one per variant without the final newline"""
    width, nlines, off, _ = FAMILIES[family]
    out = []
    fseed = 100 * list(FAMILIES).index(family)
    recs = [record("u%d_%s_%s_%s" % (i, family, v, e), width, nlines, e, v, True, seed=fseed + i)
            for i, (v, e) in enumerate(variants(True))]
    at = lambda i, r, pos: _next_edge(pos, r, 0 if r.variant == "kib" else off(r.Ln))
    data, anchors = place_records(recs, at)
    out.append(Layout("%s_nl" % family, data, recs, anchors, [path_of(v, family) for v, _ in variants(True)], family))
    for i, (v, e) in enumerate(variants(False)):
        r = record("t%d_%s_%s_%s" % (i, family, v, e), width, nlines, e, v, False, seed=fseed + 50 + i)
        data, anchors = place_records([r], at)
        out.append(Layout("%s_eof_%s_%s" % (family, v, e), data, [r], anchors, [path_of(v, family)], family))
    return out


def block_layout(shift, variant):
    """one record (LF, 80-column lines) whose last newline is at 8 MiB + shift"""
    r = record("b_%d_%s" % (shift, variant), 80, 60, "lf", variant, True, seed=abs(shift) + (7 if variant == "plus1" else 0))
    start = (BLOCK_BYTES - 4 * E.WINDOW) // (4 * E.WINDOW) * (4 * E.WINDOW)
    data, anchors = place_records([r], lambda i, r, pos: BLOCK_BYTES + shift, start=start)
    return Layout("block%+d_%s" % (shift, variant), data, [r], anchors, ["block"], "block")


@functools.lru_cache(maxsize=None)
def layouts():
    """every layout but the block ones, by name"""
    out = {}
    for fam in FAMILIES:
        for lay in family_layouts(fam):
            out[lay.name] = lay
    return out


def block_keys():
    return [(d, v) for d in BLOCK_SHIFTS for v in ("minus1", "plus1")]


# ---- the first record of a shard ----------------------------------------------------------------------------------
SHARD_WORLDS = (2, 3, 5)


@functools.lru_cache(maxsize=None)
def shard_layout():
    """records of every variant (60-column lines, and 3000-column lines whose last newline lies past region 1), back
    to back after a short lead record -> (data, recs, header offsets of recs)"""
    recs = [record("s%d_%s_%s" % (i, v, e), 60, 40, e, v, True, seed=500 + i) for i, (v, e) in enumerate(variants(True))]
    recs += [record("w%d_%s_%s" % (i, v, e), 3000, 3, e, v, True, seed=700 + i)
             for i, (v, e) in enumerate(variants(True)) if v in ("minus1", "plus1", "kib", "cancel")]
    lead = b">lead x\nACGTACGTAC\nACGT\n"
    starts = np.cumsum([len(lead)] + [len(r.data) for r in recs])[:-1]
    return lead + b"".join(r.data for r in recs), recs, [int(x) for x in starts]


def shard_cuts(world):
    """cut sets of a world: world - 1 consecutive records per set, so that every record starts a shard in one of them"""
    _, recs, starts = shard_layout()
    out = []
    for j in range(0, len(recs), world - 1):
        c = starts[j:j + world - 1]
        out.append(c if len(c) == world - 1 else starts[-(world - 1):])
    return out


# ---- the path a line takes, from the bytes ------------------------------------------------------------------------
def settled_by(data, p):
    """the path that raises the event of the line ending in the newline at p (p = len(data): the virtual one)"""
    nl, facts, k = E.region_view(data, p)
    path = E.region_path("fasta", nl, facts)
    if path != "fast":
        return path
    if k >= 2:
        return "fact"
    r = min(p, len(data)) // REGION
    if r == 0:
        return "carry"
    pnl, _, _ = E.region_view(data, (r - 1) * REGION)
    return "carry" if pnl < 2 or pnl > SEGCAP else "rows01"


# ---- a plain restatement of the bit -------------------------------------------------------------------------------
def uniform_bits(data):
    """pad[0] of every record by numpy on the bytes: the sequence-line lengths (len + 1, the unterminated last line of
    the file counted with its virtual newline) of each record; uniform iff all but the last equal the first and the
    last is no longer.  Lines before the first header belong to no record."""
    a = np.frombuffer(data, np.uint8)
    n = a.size
    ends = np.flatnonzero(a == 10)
    if n and a[-1] != 10:
        ends = np.append(ends, n)
    starts = np.concatenate([[0], ends[:-1] + 1])
    hdr = (ends > starts) & (a[np.minimum(starts, n - 1)] == ord(">")) if n else np.zeros(0, bool)
    L = ends - starts + 1
    out = []
    h = np.flatnonzero(hdr)
    for i, k in enumerate(h):
        stop = h[i + 1] if i + 1 < h.size else L.size
        ln = L[k + 1:stop]
        out.append(1 if ln.size <= 1 or (bool((ln[:-1] == ln[0]).all()) and ln[-1] <= ln[0]) else 0)
    return np.array(out, np.uint8)


def windows(rec_row, rec):
    """[s, e) windows of one record: crossing into, inside and ending at its last line, and 16 .. 4096 bytes ending at
    the record's end or around the last line break, the whole record"""
    slen = int(rec_row["slen"])
    a = rec.last_start
    out = {(0, slen), (max(0, a - 5), slen), (a, slen), (max(0, a - 1), a + 1), (a + 1, max(a + 2, slen - 1))}
    for L in (16, 17, 31, 100, 1000, 1024, 2049, 4096):
        out.add((max(0, slen - L), slen))
        out.add((max(0, a - L // 2), min(slen, a - L // 2 + L)))
        out.add((max(0, slen - L - 3), max(0, slen - 3)))
    return sorted((s, e) for s, e in out if 0 <= s < e <= slen)

