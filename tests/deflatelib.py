"""A DEFLATE (RFC 1951) writer that builds streams by hand, and a catalogue of the shapes the GPU decoder
(pyfastx_b200/csrc/fxg_inflate_core.cuh) must get right or reject.

zlib's deflate never emits most of these: a one-bit distance code, 15-bit codes, empty stored blocks, blocks of
every type at every bit phase, length 258 written as 284 + 31, and the malformed streams, one per rejection path of
the decoder.  Every catalogue entry is pinned to zlib's verdict by tests/test_deflate_streams_cpu.py.

Plain Python, no dependencies."""
import bisect
import heapq
import random
import struct
import zlib
from dataclasses import dataclass, field

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8           # RFC 1951 3.2.6, symbols 0..287
FIXED_DIST = [5] * 32                                               # symbols 30 and 31 are never valid

# decoder status codes (fxi::INF_*)
INF_BAD_BLOCK, INF_BAD_CODE, INF_OVERRUN, INF_SIZE = 2, 3, 4, 5


@dataclass(frozen=True)
class Match:
    """a back-reference, encoded with the shortest length / distance symbol that covers it"""
    length: int
    dist: int


@dataclass(frozen=True)
class Sym:
    """an explicit length symbol (257..287) with its extra bits, and an optional distance symbol (0..31) with its
    extra bits; symbols outside the RFC's tables carry no extra bits"""
    lsym: int
    lext: int = 0
    dsym: int = None
    dext: int = 0


def length_symbol(n):
    if n == 258:
        return 285, 0
    i = bisect.bisect_right(LEN_BASE, n) - 1
    return 257 + i, n - LEN_BASE[i]


def dist_symbol(d):
    i = bisect.bisect_right(DIST_BASE, d) - 1
    return i, d - DIST_BASE[i]


def canonical(lengths):
    """RFC 1951 3.2.2: the canonical code of every symbol, (code, length), or None for length 0"""
    count = [0] * 16
    for n in lengths:
        if n:
            count[n] += 1
    nxt, code = [0] * 16, 0
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    out = []
    for n in lengths:
        if n:
            out.append((nxt[n], n))
            nxt[n] += 1
        else:
            out.append(None)
    return out


def complete_lengths(nsym):
    """lengths of a complete code over nsym >= 2 symbols: k of them one bit shorter than the rest"""
    L = max(1, (nsym - 1).bit_length())
    k = (1 << L) - nsym
    return [L - 1] * k + [L] * (nsym - k)


def huffman_lengths(freq, maxbits=15):
    """Huffman code lengths for {symbol: count}; a complete code whenever two or more symbols are used (a flat
    one when the tree is deeper than maxbits), and a single one-bit code for a single symbol"""
    syms = sorted(s for s, c in freq.items() if c)
    if len(syms) == 1:
        return {syms[0]: 1}
    heap = [(freq[s], i, [s]) for i, s in enumerate(syms)]
    heapq.heapify(heap)
    depth = dict.fromkeys(syms, 0)
    tie = len(syms)
    while len(heap) > 1:
        a, _, sa = heapq.heappop(heap)
        b, _, sb = heapq.heappop(heap)
        for s in sa + sb:
            depth[s] += 1
        heapq.heappush(heap, (a + b, tie, sa + sb))
        tie += 1
    if max(depth.values()) > maxbits:
        return dict(zip(syms, complete_lengths(len(syms))))
    return depth


def rle_lengths(lens):
    """code-length symbols for a list of code lengths: (symbol, extra bits), with runs as 16 / 17 / 18"""
    out, i = [], 0
    while i < len(lens):
        v, j = lens[i], i
        while j < len(lens) and lens[j] == v:
            j += 1
        run = j - i
        if v == 0:
            while run >= 11:
                r = min(run, 138); out.append((18, r - 11)); run -= r
            if run >= 3:
                out.append((17, run - 3)); run = 0
            out += [(0, 0)] * run
        else:
            out.append((v, 0)); run -= 1
            while run >= 3:
                r = min(run, 6); out.append((16, r - 3)); run -= r
            out += [(v, 0)] * run
        i = j
    return out


class Writer:
    """bits LSB first, Huffman codes MSB first (RFC 1951 3.1.1); `data` is what a decoder that follows the
    symbols as written produces (for malformed streams: what the trailer's CRC and ISIZE then describe)"""

    def __init__(self):
        self.buf, self.acc, self.nacc = bytearray(), 0, 0
        self.data = bytearray()

    @property
    def nbits(self):
        return 8 * len(self.buf) + self.nacc

    def bits(self, value, n):
        assert 0 <= value < (1 << n) or (n == 0 and value == 0), (value, n)
        self.acc |= value << self.nacc
        self.nacc += n
        while self.nacc >= 8:
            self.buf.append(self.acc & 255)
            self.acc >>= 8
            self.nacc -= 8

    def code(self, c):
        code, n = c
        self.bits(int(format(code, "0%db" % n)[::-1], 2), n)

    def align(self):
        if self.nacc:
            self.buf.append(self.acc)
            self.acc, self.nacc = 0, 0

    def getvalue(self):
        return bytes(self.buf) + (bytes([self.acc]) if self.nacc else b"")

    # ---- blocks ----
    def stored(self, payload, last=False, nlen=None, present=None):
        """a stored block; `nlen` overrides NLEN, `present` cuts the payload that is actually written"""
        self.bits(int(last), 1)
        self.bits(0, 2)
        self.align()
        self.bits(len(payload), 16)
        self.bits(len(payload) ^ 0xffff if nlen is None else nlen, 16)
        self.buf += payload[:present]
        self.data += payload

    def fixed(self, symbols, last=False, eob=True):
        self.bits(int(last), 1)
        self.bits(1, 2)
        self._symbols(symbols, canonical(FIXED_LIT), canonical(FIXED_DIST), eob)

    def dynamic(self, symbols, last=False, lit_lens=None, dist_lens=None, cl_lens=None, cl_syms=None, hclen=None,
                eob=True):
        """a dynamic block.  Without lit_lens / dist_lens the codes are Huffman codes of the symbols used (an
        all-zero distance code when there are no matches); without cl_syms the code lengths are run-length coded
        with 16 / 17 / 18; without cl_lens the code-length code is a Huffman code of the symbols cl_syms uses"""
        if lit_lens is None or dist_lens is None:
            lf, df = {256: 1}, {}
            for s in symbols:
                ls, ds = self._parts(s)
                lf[ls] = lf.get(ls, 0) + 1
                if ds is not None:
                    df[ds] = df.get(ds, 0) + 1
            if lit_lens is None:
                h = huffman_lengths(lf)
                lit_lens = [h.get(i, 0) for i in range(max(257, max(h) + 1))]
            if dist_lens is None:
                h = huffman_lengths(df) if df else {}
                dist_lens = [h.get(i, 0) for i in range(max(h) + 1)] if h else [0]
        if cl_syms is None:
            cl_syms = rle_lengths(list(lit_lens) + list(dist_lens))
        if cl_lens is None:
            cf = {}
            for s, _ in cl_syms:
                cf[s] = cf.get(s, 0) + 1
            h = huffman_lengths(cf, 7)
            if len(h) == 1:                      # the code-length code must be complete: add a second code
                h[18 if 18 not in h else 0] = 1
            cl_lens = [h.get(i, 0) for i in range(19)]
        if hclen is None:
            hclen = max(4, max(i + 1 for i in range(19) if cl_lens[CL_ORDER[i]]))
        self.bits(int(last), 1)
        self.bits(2, 2)
        self.bits(len(lit_lens) - 257, 5)
        self.bits(len(dist_lens) - 1, 5)
        self.bits(hclen - 4, 4)
        for i in range(hclen):
            self.bits(cl_lens[CL_ORDER[i]], 3)
        cc = canonical(cl_lens)
        for s, x in cl_syms:
            self.code(cc[s])
            if s >= 16:
                self.bits(x, {16: 2, 17: 3, 18: 7}[s])
        self._symbols(symbols, canonical(lit_lens), canonical(dist_lens), eob)

    @staticmethod
    def _parts(s):
        if isinstance(s, int):
            return s, None
        if isinstance(s, Match):
            return length_symbol(s.length)[0], dist_symbol(s.dist)[0]
        return s.lsym, s.dsym

    def _symbols(self, symbols, lc, dc, eob):
        for s in symbols:
            if isinstance(s, int):
                self.code(lc[s])
                self.data.append(s)
                continue
            if isinstance(s, Match):
                ls, lx = length_symbol(s.length)
                ds, dx = dist_symbol(s.dist)
                s = Sym(ls, lx, ds, dx)
            self.code(lc[s.lsym])
            if s.lsym - 257 < 29:
                self.bits(s.lext, LEN_EXTRA[s.lsym - 257])
            if s.dsym is None:
                continue
            self.code(dc[s.dsym])
            if s.dsym < 30:
                self.bits(s.dext, DIST_EXTRA[s.dsym])
            if s.lsym - 257 < 29 and s.dsym < 30:
                n = LEN_BASE[s.lsym - 257] + s.lext
                d = DIST_BASE[s.dsym] + s.dext
                for _ in range(n):
                    self.data.append(self.data[-d] if d <= len(self.data) else 0)
        if eob:
            self.code(lc[256])


# ---- gzip / BGZF members ----------------------------------------------------------------------------------------
def gzip_member(deflate, data, isize=None, junk=b"", fname=None, comment=None, fhcrc=False, extra=b"", bgzf=True):
    """a gzip member (RFC 1952) around raw deflate bytes: CRC-32 and ISIZE of `data` (ISIZE overridable), `junk`
    between the deflate data and the trailer.  BGZF: a 'BC' subfield (SAM spec 4.1) after the caller's `extra`
    subfields; a member over 64 KiB, which BGZF cannot describe, gets BSIZE 0xffff."""
    flg = (4 if bgzf or extra else 0) | (8 if fname is not None else 0) | (16 if comment is not None else 0) | (2 if fhcrc else 0)
    xfield = extra + (b"BC\x02\x00\x00\x00" if bgzf else b"")
    tail = b""
    if fname is not None:
        tail += fname + b"\x00"
    if comment is not None:
        tail += comment + b"\x00"
    total = 10 + (2 + len(xfield) if flg & 4 else 0) + len(tail) + (2 if fhcrc else 0) + len(deflate) + len(junk) + 8
    if bgzf:
        xfield = xfield[:-2] + struct.pack("<H", min(total - 1, 0xffff))
    hdr = b"\x1f\x8b\x08" + bytes([flg]) + b"\x00\x00\x00\x00\x00\xff"
    if flg & 4:
        hdr += struct.pack("<H", len(xfield)) + xfield
    hdr += tail
    if fhcrc:
        hdr += struct.pack("<H", zlib.crc32(hdr) & 0xffff)
    return hdr + deflate + junk + struct.pack("<II", zlib.crc32(data), len(data) if isize is None else isize)


BGZF_EOF = gzip_member(b"\x03\x00", b"")


@dataclass
class Stream:
    """one catalogue entry: raw deflate bytes and the bytes they decode to, or out=None for a stream zlib rejects.
    `data` is what the symbols as written spell out (the trailer's CRC-32 and, unless `isize` says otherwise, its
    ISIZE); `status` is the decoder's INF_* code for a rejected stream (None: any nonzero)"""
    name: str
    deflate: bytes
    out: bytes
    data: bytes = None
    status: int = None
    isize: int = None
    junk: bytes = b""
    header: dict = field(default_factory=dict)

    def __post_init__(self):
        if self.data is None:
            self.data = self.out

    def member(self, bgzf=True):
        return gzip_member(self.deflate, self.data, isize=self.isize, junk=self.junk, bgzf=bgzf, **self.header)


def _w():
    return Writer()


def _valid(name, w, **kw):
    return Stream(name, w.getvalue(), bytes(w.data), **kw)


def _invalid(name, w, status, **kw):
    return Stream(name, w.getvalue(), None, data=bytes(w.data), status=status, **kw)


def lits(b):
    return list(b)


def window_edge_stream(seed=5):
    """40,000 stored bytes, then a block whose first symbol is a match at distance 32,768: a checkpoint placed
    at that block (32 KiB spacing) starts a segment whose first match reads byte 0 of the checkpoint's window"""
    rng = random.Random(seed)
    w = _w()
    w.stored(bytes(rng.randrange(256) for _ in range(40000)))
    w.fixed([Match(258, 32768), Match(77, 32768)] + lits(b"edge") + [Match(40, 32767), Match(3, 1)], last=True)
    return _valid("window_edge", w)


def catalogue():
    rng = random.Random(20261017)
    text = b"the decoder must agree with zlib on every stream, valid or not. " * 3
    acgt = bytes(rng.choice(b"ACGT") for _ in range(300))
    C = []

    # ---- valid ----
    w = _w(); w.stored(text, last=True); C.append(_valid("stored_only", w))
    w = _w(); w.fixed(lits(acgt[:40]) + [Match(20, 8), Match(258, 1)] + lits(b"xyz"), last=True); C.append(_valid("fixed_only", w))
    w = _w(); w.dynamic(lits(text[:64]) + [Match(64, 64), Match(100, 37)] + lits(acgt[:50]), last=True); C.append(_valid("dynamic_only", w))
    for p in range(8):
        # a fixed block that leaves the next block header at bit phase p: 3 + 7 header / EOB bits plus one extra bit
        # per 9-bit literal (144..255)
        w = _w()
        w.fixed(lits(b"AC") + [200] * ((p - 2) % 8))
        assert w.nbits % 8 == p
        w.stored(acgt[:33 + p])
        w.dynamic(lits(text[:20 + p]) + [Match(11 + p, 20)])
        w.fixed([150 + p, Match(5, 3)])
        w.stored(b"", last=True)
        C.append(_valid("mixed_phase%d" % p, w))
    w = _w(); w.stored(b""); w.fixed(lits(b"after an empty stored block"), last=True); C.append(_valid("stored_empty", w))
    w = _w(); w.stored(bytes(rng.randrange(256) for _ in range(65535)), last=True); C.append(_valid("stored_65535", w))
    w = _w(); w.dynamic(lits(range(256)) + [Match(258, 256)] * 253 + [Match(6, 256)], last=True)
    assert len(w.data) == 65536
    C.append(_valid("output_65536", w))
    # 15-bit literal codes: lengths 1..14, 15, 15 over 16 symbols (complete); 'O' and EOB are 15 bits long
    ll = [0] * 257
    for i, n in enumerate(range(1, 15)):
        ll[65 + i] = n
    ll[65 + 14] = 15; ll[256] = 15
    w = _w(); w.dynamic(lits(b"ONAO" * 300), lit_lens=ll, dist_lens=[0], last=True); C.append(_valid("lit_codes_15_bits", w))
    # 15-bit distance codes: symbol 7 (distances 13..16) takes one of the two 15-bit codes
    dl = [0] * 30
    for i, n in enumerate(list(range(1, 15)) + [15, 15]):
        dl[i] = n
    dl[7], dl[14] = dl[14], dl[7]
    w = _w(); w.dynamic(lits(b"ABCDEFGHIJKLMNOP") + [Match(3, 16)] * 500 + [Match(4, 2)], lit_lens=[9] * 256 + [3, 3, 3, 3],
                        dist_lens=dl, last=True)
    C.append(_valid("dist_codes_15_bits", w))
    w = _w(); w.dynamic(lits(b"G") + [Match(30, 1)], lit_lens=[9] * 256 + [2] + [0] * 14 + [2],
                        dist_lens=[1], last=True)
    C.append(_valid("dist_code_single_1_bit", w))
    w = _w(); w.dynamic(lits(text[:40]), dist_lens=[0], last=True); C.append(_valid("dist_code_all_zero", w))
    w = _w(); w.dynamic([], lit_lens=[0] * 256 + [1], dist_lens=[0], last=True); C.append(_valid("lit_code_single_eob", w))
    # every length 3..258 at every distance 1..32, overlapping when length > distance
    syms = lits(acgt[:32]) + [Match(n, 1 + (n % 32)) for n in range(3, 259)]
    w = _w(); w.fixed(syms, last=True); C.append(_valid("overlap_fixed", w))
    w = _w(); w.dynamic(lits(acgt[32:64]) + [Match(n, 1 + ((n * 7) % 32)) for n in range(258, 2, -1)], last=True)
    C.append(_valid("overlap_dynamic", w))
    w = _w(); w.fixed(lits(b"A") + [Sym(284, 31, 0, 0)], last=True)
    assert len(w.data) == 259
    C.append(_valid("len_284_plus_31", w))
    w = _w(); w.fixed(lits(acgt[:100]) + [Match(50, 100)], last=True); C.append(_valid("dist_equals_output", w))
    w = _w(); w.stored(bytes(rng.randrange(256) for _ in range(32768))); w.fixed([Match(258, 32768), Match(100, 32768)], last=True)
    C.append(_valid("dist_32768", w))
    w = _w(); w.fixed([], last=True); C.append(_valid("empty_fixed", w))
    w = _w(); w.stored(b"", last=True); C.append(_valid("empty_stored", w))
    C.append(window_edge_stream())
    small = _w(); small.fixed(lits(b"header variants ") + [Match(16, 16)], last=True)
    for name, hdr in [("hdr_fname", dict(fname=b"reads.fq")), ("hdr_comment", dict(comment=b"a comment")),
                      ("hdr_fhcrc", dict(fhcrc=True)), ("hdr_extra_before_bc", dict(extra=b"XY\x03\x00abcZZ\x00\x00")),
                      ("hdr_all", dict(fname=b"n", comment=b"", fhcrc=True, extra=b"AB\x01\x00q"))]:
        C.append(_valid(name, small, header=hdr))

    # ---- rejected: one entry per rejection path ----
    w = _w(); w.bits(1, 1); w.bits(3, 2); C.append(_invalid("btype_3", w, INF_BAD_BLOCK))
    w = _w(); w.stored(b"abc", last=True, nlen=0xfffd); C.append(_invalid("stored_nlen_mismatch", w, INF_BAD_BLOCK))
    w = _w(); w.dynamic(lits(b"A"), lit_lens=complete_lengths(287), dist_lens=[1], last=True); C.append(_invalid("hlit_287", w, INF_BAD_BLOCK))
    w = _w(); w.dynamic(lits(b"A"), lit_lens=[9] * 256 + [3, 3, 3, 3], dist_lens=[5] * 31, last=True); C.append(_invalid("hdist_31", w, INF_BAD_BLOCK))
    lens = [9] * 256 + [3, 3, 3, 3] + [1]
    w = _w(); w.dynamic(lits(b"A"), lit_lens=lens[:-1], dist_lens=[1], cl_syms=[(16, 0)] + rle_lengths(lens), last=True)
    C.append(_invalid("repeat_16_first", w, INF_BAD_CODE))
    w = _w(); w.dynamic(lits(b"A"), lit_lens=lens[:-1], dist_lens=[1, 0, 0, 0, 0], cl_syms=rle_lengths(lens) + [(17, 7)], last=True)
    C.append(_invalid("repeat_past_hlit_hdist", w, INF_BAD_CODE))
    # EOB is the longest code: the zero padding decodes as literals, and the stream runs on into the trailer
    w = _w(); w.dynamic(lits(b"AAAAAAAAAC"), lit_lens=[0] * 65 + [1, 0, 2] + [0] * 188 + [2], dist_lens=[0], last=True, eob=False)
    C.append(_invalid("missing_eob", w, None))
    w = _w(); w.dynamic(lits(b"AB"), lit_lens=[0] * 65 + [1, 1] + [0] * 189 + [1], dist_lens=[0], last=True, eob=False)
    C.append(_invalid("lit_code_oversubscribed", w, INF_BAD_CODE))
    w = _w(); w.dynamic(lits(b"AB") + [Match(3, 1)], lit_lens=[9] * 256 + [3, 3, 3, 3], dist_lens=[1, 1, 1], last=True)
    C.append(_invalid("dist_code_oversubscribed", w, INF_BAD_CODE))
    # the four shapes zlib rejects although the bytes and the trailer agree
    w = _w(); w.dynamic(lits(b"ACA"), lit_lens=[0] * 65 + [2, 0, 2] + [0] * 188 + [2], dist_lens=[1], last=True)
    C.append(_invalid("lit_code_incomplete", w, INF_BAD_CODE))
    w = _w(); w.dynamic(lits(b"A") + [Match(3, 1)], lit_lens=[9] * 256 + [3, 3, 3, 3], dist_lens=[2, 2], last=True)
    C.append(_invalid("dist_code_incomplete", w, INF_BAD_CODE))
    one = [0] * 65 + [1] + [0] * 190 + [1]
    plain = [(n, 0) for n in one + [1]]                          # code lengths without run symbols
    w = _w(); w.dynamic(lits(b"A"), lit_lens=one, dist_lens=[1], cl_lens=[4] * 19, cl_syms=plain, last=True)
    C.append(_invalid("cl_code_oversubscribed", w, INF_BAD_CODE))
    w = _w(); w.dynamic(lits(b"A"), lit_lens=one, dist_lens=[1], cl_lens=[5] * 16 + [0, 0, 0], cl_syms=plain, last=True)
    C.append(_invalid("cl_code_incomplete", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(acgt[:30]) + [Match(12, 4)], last=True); C.append(_invalid("junk_before_trailer", w, INF_BAD_BLOCK, junk=b"\x00"))
    w = _w(); w.stored(acgt[:30], last=True); C.append(_invalid("junk_after_stored", w, INF_BAD_BLOCK, junk=b"\x00\x00\x00"))
    w = _w(); w.fixed(lits(b"AB") + [Sym(286)], last=True); C.append(_invalid("fixed_lit_286", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(b"AB") + [Sym(287)], last=True); C.append(_invalid("fixed_lit_287", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(b"AB") + [Sym(257, 0, 30)], last=True); C.append(_invalid("fixed_dist_30", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(b"AB") + [Sym(257, 0, 31)], last=True); C.append(_invalid("fixed_dist_31", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(b"ABC") + [Match(3, 4)], last=True); C.append(_invalid("dist_past_member_start", w, INF_BAD_CODE))
    w = _w(); w.fixed(lits(text[:50]), last=True); C.append(_invalid("output_longer_than_isize", w, INF_OVERRUN, isize=49))
    w = _w(); w.fixed(lits(text[:50]), last=True); C.append(_invalid("output_shorter_than_isize", w, INF_SIZE, isize=51))
    w = _w(); w.stored(text[:100], last=True, present=60); C.append(_invalid("truncated_stored", w, INF_OVERRUN))
    w = _w(); w.dynamic(lits(text[:120]), last=True)
    C.append(Stream("truncated_dynamic", w.getvalue()[:-6], None, data=bytes(w.data)))
    return C


def zlib_verdict(s):
    """zlib's answer for a catalogue entry: the bytes of its gzip member (header, data, CRC-32 and ISIZE all
    checked: wbits=31), or None when zlib raises"""
    try:
        d = zlib.decompressobj(31)
        out = d.decompress(s.member(bgzf=False))
        if not d.eof or d.unused_data:
            return None
        return out
    except zlib.error:
        return None


def pack_members(members):
    """gzip members laid end to end -> (bytes, compressed offsets, uncompressed offsets from each ISIZE), n + 1
    entries each; offsets are computed here, not by walking BGZF headers, so members over 64 KiB fit too"""
    co, uo = [0], [0]
    for m in members:
        co.append(co[-1] + len(m))
        uo.append(uo[-1] + struct.unpack("<I", m[-4:])[0])
    return b"".join(members), co, uo
