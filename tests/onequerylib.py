"""Inputs and expected answers of the one-query getters (fa[name][s:e].seq, fq[i].seq / .qual ...) for
test_one_query_gpu.py and test_one_query_cpu.py.

fxg_extract_one_host / fxg_read_one_host (csrc/fxg_extract.cu) choose a path from the query's length: the resident
service kernel up to SVC_LIMIT bytes, else one launch of extract_one_kernel / read_one_kernel that writes to mapped
pinned memory up to ONE_PINNED bytes and to a device buffer beyond.  extract_one_kernel cuts a query of a splittable
record into pieces of at least PIECE bytes, at most sm_count * CTAS_PER_SM * XWARPS of them, so past
sm_count * CTAS_PER_SM * XWARPS * PIECE bytes every piece grows.  test_one_query_cpu.py checks these constants against
the source, and every layout and schedule here against the oracle."""
import numpy as np

from oracle import fxo

SVC_LIMIT = 65536            # longest query the service kernel takes
ONE_PINNED = 1 << 20         # longest query written straight to mapped pinned memory
PIECE = 2048                 # bytes per warp below which extract_one_kernel does not split further
XWARPS = 8                   # warps per CTA of the one-query kernels
CTAS_PER_SM = 4              # extract_one_kernel: at most sm_count * CTAS_PER_SM * XWARPS pieces
BIG_SLICE = 40_000_007       # the ~40 MB slice
NOMINAL_SMS = 132            # H100 SXM; the CPU companion builds the layouts for this count

UPPER, REVERSE, COMPLEMENT = fxo.UPPER, fxo.REVERSE, fxo.COMPLEMENT
RC = REVERSE | COMPLEMENT
GETTERS = {0: "seq", REVERSE: "reverse", COMPLEMENT: "complement", RC: "antisense"}
IUPAC = np.frombuffer(b"RYKMSWBDHVN", np.uint8)


def threshold(sm_count):
    """query length past which extract_one_kernel's pieces grow beyond PIECE bytes"""
    return sm_count * CTAS_PER_SM * XWARPS * PIECE


def fasta_lengths(sm_count):
    t = threshold(sm_count)
    return [1, 15, 16, 17, 2047, 2048, 2049, 16383, 16384, 16385, 65535, 65536, 65537,
            (1 << 20) - 1, 1 << 20, (1 << 20) + 1, t - 16, t, t + 1, t + 16]


FASTQ_LENGTHS = [1, 150, 65535, 65536, 65537, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, 3 << 20]


def path_of(n):
    """'service' | 'mapped' | 'device': where a query of n bytes is served with the service on"""
    return "service" if n <= SVC_LIMIT else ("mapped" if n <= ONE_PINNED else "device")


def residues(n, rng):
    """n sequence bytes: A/C/G/T with about 1 % IUPAC letters, in soft-masked (lower case) runs of a few hundred"""
    a = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n)]
    iu = rng.random(n) < 0.01
    a[iu] = IUPAC[rng.integers(0, IUPAC.size, int(iu.sum()))]
    lower = (np.cumsum(rng.random(n) < 1 / 300) & 1).astype(bool)
    a[lower] |= 0x20
    return a


def fasta_record(name, seq, width, eol=b"\n", last=None, blank_after=None, trailing=True):
    """header + sequence lines of `width` bytes; `last` bytes of the sequence go on one final line of their own (a longer
    last line); a blank line after line `blank_after`; no end of line after the last line if not `trailing`"""
    body, tail = (seq, None) if last is None else (seq[:-last], seq[-last:])
    n_full = body.size // width
    full = body[:n_full * width].reshape(n_full, width)
    e = np.frombuffer(eol, np.uint8)
    lines = np.concatenate([full, np.broadcast_to(e, (n_full, e.size))], axis=1).ravel().tobytes()
    if blank_after is not None:
        k = blank_after * (width + e.size)
        lines = lines[:k] + eol + lines[k:]
    rest = body[n_full * width:].tobytes()
    if rest:
        lines += rest + eol
    if tail is not None:
        lines += tail.tobytes() + eol
    if not trailing:
        assert lines.endswith(eol)
        lines = lines[:-len(eol)]
    return b">" + name.encode() + b" layout" + eol + lines


def fasta_layouts(sm_count, seed=1):
    """(file bytes, layouts): records with the layouts the one-query paths treat differently, in one file.
    layouts[i] = dict(name, norm, uniform, lengths) for record i; lengths = the query lengths it is asked for."""
    rng = np.random.default_rng(seed)
    t = threshold(sm_count)
    lens = fasta_lengths(sm_count)
    small = [n for n in lens if n <= (1 << 20) + 1]
    specs = [
        # name, slen, record kwargs, norm, uniform, lengths
        ("lf60", BIG_SLICE + 6_000_033, dict(width=60), 1, 1, lens + [BIG_SLICE]),
        ("crlf80", t + 350_011, dict(width=80, eol=b"\r\n"), 1, 1, lens),
        ("longlast", 3_000_023, dict(width=60, last=200_003), 1, 0, small),
        ("blank", 3_000_029, dict(width=60, blank_after=20_000), 0, 0, small),
        ("oneline", 5_000_011, dict(width=5_000_011), 1, 1, small),
        ("tail", 1_300_021, dict(width=60, trailing=False), 1, 1, small),
    ]
    data, layouts = [], []
    for name, slen, kw, norm, uniform, qlens in specs:
        data.append(fasta_record(name, residues(slen, rng), **kw))
        layouts.append(dict(name=name, slen=slen, norm=norm, uniform=uniform, lengths=sorted(set(qlens + [slen]))))
    return b"".join(data), layouts


def starts(slen, n):
    """0, slen - n and an odd offset in the middle"""
    return sorted({0, slen - n, min(((slen - n) // 2) | 1, slen - n)})


def fasta_queries(layouts, rows):
    """(row, s, e, flags) of every record, length, start and flag combination (upper x the four getters)"""
    q = []
    for i, lay in enumerate(layouts):
        slen = int(rows["slen"][i])
        for n in lay["lengths"]:
            for s in starts(slen, n):
                for f in (0, REVERSE, COMPLEMENT, RC, UPPER, UPPER | REVERSE, UPPER | COMPLEMENT, UPPER | RC):
                    q.append((i, s, s + n, f))
    return q


def quals(n, rng):
    """n quality bytes over the whole printable range 33..126"""
    return rng.integers(33, 127, n).astype(np.uint8)


def fastq_file(lengths, eol=b"\n", trailing=True, seed=2):
    """reads of the given lengths (IUPAC letters, soft-masked runs, qualities 33..126); no end of line after the last
    quality line if not `trailing`"""
    rng = np.random.default_rng(seed)
    out = []
    for k, n in enumerate(lengths):
        out.append(b"@r%d len=%d" % (k, n) + eol + residues(n, rng).tobytes() + eol + b"+" + eol +
                   quals(n, rng).tobytes() + eol)
    data = b"".join(out)
    return data if trailing else data[:-len(eol)]


_LUT = None


def transform(b, flags):
    """upper case, complement (fxo.complement_lut) and reverse of a read's bytes, as the read getters apply them"""
    global _LUT
    if _LUT is None:
        _LUT = fxo.complement_lut()
    a = np.frombuffer(b, np.uint8)
    if flags & UPPER:
        a = np.where((a >= 97) & (a <= 122), a - 32, a).astype(np.uint8)
    if flags & COMPLEMENT:
        a = _LUT[a]
    if flags & REVERSE:
        a = a[::-1]
    return a.tobytes()


def read_expected(data, row, which, flags):
    """oracle bytes of one read's sequence (which = 0) or quality (which = 1) under `flags`: qualities are only ever
    reversed, never upper-cased or complemented"""
    sq, ql = fxo.read_fetch(data, row)
    return transform(sq, flags) if which == 0 else transform(ql, flags & REVERSE)


def schedule(n_calls, fasta_sets, fastq_set, seed=7):
    """a seeded list of getter calls that switches between objects, between FASTA and FASTQ and between the service,
    mapped-launch and device-buffer paths from one call to the next.
    fasta_sets: {key: (slens, upper)}; fastq_set: rlens.  Items: ("fa", key, row, s, e, getter flags) or
    ("fq", row, which, flags).  Lengths cycle through the three paths so that no two consecutive calls share one."""
    rng = np.random.default_rng(seed)
    keys = sorted(fasta_sets)
    fq_rlens = np.asarray(fastq_set)
    by_path = {p: [i for i, n in enumerate(fq_rlens) if path_of(int(n)) == p] for p in ("service", "mapped", "device")}
    out = []
    paths = ("service", "mapped", "service", "device")
    for k in range(n_calls):
        want = paths[k % len(paths)]
        if k % 3 == 2 and by_path[want]:
            i = int(rng.choice(by_path[want]))
            which = int(rng.integers(0, 2))
            out.append(("fq", i, which, 0 if which else int(rng.choice([0, REVERSE, COMPLEMENT, RC]))))
            continue
        key = keys[int(rng.integers(0, len(keys)))]
        slens, _ = fasta_sets[key]
        i = int(rng.integers(0, len(slens)))
        slen = int(slens[i])
        lo, hi = {"service": (1, SVC_LIMIT), "mapped": (SVC_LIMIT + 1, ONE_PINNED),
                  "device": (ONE_PINNED + 1, 3 * ONE_PINNED)}[want]
        hi = min(hi, slen)
        if lo > hi:
            lo, hi = 1, min(SVC_LIMIT, slen)
        n = int(rng.integers(lo, hi + 1))
        s = int(rng.integers(0, slen - n + 1))
        out.append(("fa", key, i, s, s + n, int(rng.choice([0, REVERSE, COMPLEMENT, RC]))))
    return out


PINNED_CHUNK = 256 << 20     # pageable uploads are staged through pinned buffers of this size
UPLOAD_QUERY = (7, 7 + 60_000)


def upload_order_data():
    """-> (bytes, FASTA rows, FASTQ rows): a FASTA part larger than PINNED_CHUNK (4 MB records repeated) whose last
    record is unique, followed by three FASTQ reads; the rows address the whole buffer"""
    rng = np.random.default_rng(9)
    block = fasta_record("fill", residues(4_000_000, rng), 60)
    fa_part = block * (PINNED_CHUNK // len(block) + 10) + fasta_record("last", residues(70_001, rng), 60)
    fq_part = fastq_file([150, 1000, 60_000], seed=10)
    frows = fxo.fasta_scan(fa_part)[0]
    qrows = fxo.fastq_scan(fq_part)[0]
    qrows["soff"] += len(fa_part)
    qrows["qoff"] += len(fa_part)
    return fa_part + fq_part, frows, qrows
