// fxg_inflate_core.cuh -- one DEFLATE (RFC 1951) member decoded by ONE thread.
//
// Used by inflate_thread_kernel (fxg_inflate.cu) with a thread per BGZF member: 32 members per warp, so the
// serial Huffman decode -- which cannot be spread over the lanes of a warp -- still fills every lane.
// The code is plain C++ (no CUDA intrinsics) so that tests/test_inflate_core_cpu.py can compile the very
// same functions for the host and check them against zlib without a GPU.  Nothing here is a CPU fallback:
// the product only calls it from the kernel.
//
// Replaces zlib's inflate() as used by gzread during the scan (reference src/kseq.c:70) and by
// zran_read per access (src/index.c:685-686).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define FXI_HD __host__ __device__ __forceinline__
#else
#define FXI_HD inline
#endif
#ifdef __CUDA_ARCH__
#define FXI_LDG32(p) __ldg(p)
#else
#define FXI_LDG32(p) (*(p))
#endif

namespace fxi {

#ifndef FXG_TL_BITS
#define FXG_TL_BITS 9
#endif
#ifndef FXG_TD_BITS
#define FXG_TD_BITS 8
#endif
constexpr int TL_BITS = FXG_TL_BITS;  // primary literal/length table: 2^TL_BITS entries (longer codes: canonical slow path)
constexpr int TD_BITS = FXG_TD_BITS;  // primary distance table

// Per-member decode tables (one member = one thread; shared memory in the kernel).  2,240 bytes.
struct MemberTables {
    uint16_t lit[1 << TL_BITS];       // (len << 9) | symbol, 0 = code longer than TL_BITS (or unused)
    uint16_t dist[1 << TD_BITS];      // (len << 5) | symbol
    uint16_t litcnt[16], litsym[288]; // canonical tables: the slow path for long codes
    uint16_t distcnt[16], distsym[32];
};
static_assert(sizeof(MemberTables) == 2 * ((1 << TL_BITS) + (1 << TD_BITS)) + 704, "MemberTables layout");

enum { INF_OK = 0, INF_BAD_HEADER = 1, INF_BAD_BLOCK = 2, INF_BAD_CODE = 3, INF_OVERRUN = 4, INF_SIZE = 5 };

struct Bits {
    const uint8_t *in;
    int64_t pos, end, lim;   // next byte to load / one past the deflate data / readable bytes at `in`
    uint64_t buf;
    int nbits;
    // at least 32 valid bits afterwards (bytes past `end` read as whatever follows, or 0 past `lim`)
    FXI_HD void refill() {
        if (nbits < 32) {
            if (pos + 8 <= lim) {
                const uint32_t *w = reinterpret_cast<const uint32_t *>(in + (pos & ~(int64_t)3));
                const uint32_t a = FXI_LDG32(w), b = FXI_LDG32(w + 1);
                const int sh = (int)(pos & 3) * 8;
                const uint32_t v = sh ? (a >> sh) | (b << (32 - sh)) : a;
                buf |= (uint64_t)v << nbits;
                nbits += 32;
                pos += 4;
            } else {
                while (nbits <= 56) {
                    const uint64_t b = pos < lim ? in[pos] : 0;
                    ++pos;
                    buf |= b << nbits;
                    nbits += 8;
                }
            }
        }
    }
    FXI_HD uint32_t peek(int n) const { return (uint32_t)(buf & ((1ull << n) - 1)); }
    FXI_HD void drop(int n) { buf >>= n; nbits -= n; }
    FXI_HD uint32_t get(int n) { refill(); const uint32_t v = peek(n); drop(n); return v; }
    FXI_HD bool overrun() const { return pos - (nbits >> 3) > end; }
};

FXI_HD uint32_t bitrev(uint32_t v, int n) {
    uint32_t r = 0;
    for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1u); v >>= 1; }
    return r;
}

// canonical decode, one bit at a time -- codes longer than the primary table
FXI_HD int slow_decode(Bits &br, const uint16_t *cnt, const uint16_t *sym) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= 15; ++len) {
        code |= (int)br.get(1);
        const int count = cnt[len];
        if (code - count < first) return sym[index + (code - first)];
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

// Primary + canonical tables for `n` symbols with code lengths lens[0..n).  False, as zlib's inflate_table decides, if
// the code is over-subscribed, or incomplete unless it is empty or a single code of length 1.
FXI_HD bool build_table(const uint8_t *lens, int n, uint16_t *tab, int tab_bits, int sym_shift, uint16_t *cnt,
                        uint16_t *sym) {
    for (int i = 0; i < 16; ++i) cnt[i] = 0;
    for (int i = 0; i < n; ++i) cnt[lens[i]]++;
    int left = 1;
    for (int len = 1; len <= 15; ++len) left = (left << 1) - cnt[len];     // once negative, stays negative
    // complete; or no code at all; or one code of length 1 (which alone leaves 2^14 of the 2^15 code space)
    const bool ok = left == 0 || left == (1 << 15) || (left == (1 << 14) && cnt[1] == 1);
    uint16_t offs[16], next[16];
    offs[1] = 0;
    for (int len = 1; len < 15; ++len) offs[len + 1] = (uint16_t)(offs[len] + cnt[len]);
    for (int i = 0; i < n; ++i)
        if (lens[i]) sym[offs[lens[i]]++] = (uint16_t)i;
    for (int i = 0; i < (1 << tab_bits); ++i) tab[i] = 0;
    if (!ok) return false;
    {
        int code = 0;
        next[0] = 0;
        for (int len = 1; len <= 15; ++len) {
            code = (code + (len > 1 ? cnt[len - 1] : 0)) << 1;
            next[len] = (uint16_t)code;
        }
    }
    // symbols are stored in `sym` grouped by length in increasing symbol order: entry k of length len has
    // code next[len] + k
    int base = 0;
    for (int len = 1; len <= tab_bits; ++len) {
        const int c = cnt[len];
        for (int k = 0; k < c; ++k) {
            const int s = sym[base + k];
            const uint32_t r = bitrev((uint32_t)(next[len] + k), len);
            const uint16_t e = (uint16_t)((len << sym_shift) | s);
            for (uint32_t j = r; j < (1u << tab_bits); j += (1u << len)) tab[j] = e;
        }
        base += c;
    }
    return true;
}

// `len` bytes from out[src..) to out[dst..), src < dst, as DEFLATE defines it (overlap repeats the pattern).
// Bytes of the source that lie before `o0` (a segment that starts at a zran checkpoint: its first matches reach back
// into the 32 KiB of output in front of the checkpoint) come from the checkpoint's window `win[0 .. wlen)`, whose last
// byte is output byte o0 - 1.
FXI_HD void copy_match(uint8_t *out, int64_t dst, int64_t src, int len, int64_t out_cap, int64_t o0 = 0,
                       const uint8_t *win = nullptr, int wlen = 0) {
    while (len > 0 && src < o0) {                     // only with a window (the BGZF path checks dist <= opos - o0)
        out[dst++] = win[wlen - (int)(o0 - src)];
        ++src; --len;
    }
    if (len <= 0) return;
    const int64_t dist = dst - src;
    while (len > 0) {
        const int n = len < 24 ? len : 24;
        if (dist >= n && (src & ~(int64_t)7) + 32 <= out_cap) {
            // no overlap within this piece: four aligned 8-byte loads issued together, stores from registers
            const uint64_t *w = reinterpret_cast<const uint64_t *>(out + (src & ~(int64_t)7));
            const uint64_t a0 = w[0], a1 = w[1], a2 = w[2], a3 = w[3];
            const int sh = (int)(src & 7) * 8;
            uint64_t v0 = a0, v1 = a1, v2 = a2;
            if (sh) {
                v0 = (a0 >> sh) | (a1 << (64 - sh));
                v1 = (a1 >> sh) | (a2 << (64 - sh));
                v2 = (a2 >> sh) | (a3 << (64 - sh));
            }
            uint8_t *o = out + dst;
            for (int i = 0; i < 8; ++i) if (i < n) o[i] = (uint8_t)(v0 >> (8 * i));
            if (n > 8) {
                for (int i = 0; i < 8; ++i) if (8 + i < n) o[8 + i] = (uint8_t)(v1 >> (8 * i));
                if (n > 16)
                    for (int i = 0; i < 8; ++i) if (16 + i < n) o[16 + i] = (uint8_t)(v2 >> (8 * i));
            }
        } else {
            for (int i = 0; i < n; ++i) out[dst + i] = out[src + i];
        }
        dst += n; src += n; len -= n;
    }
}

struct DeflateConsts {
    const uint16_t *LEN_BASE; const uint8_t *LEN_EXTRA;
    const uint16_t *DIST_BASE; const uint8_t *DIST_EXTRA;
    const uint8_t *CL_ORDER;
};

// Resumable decoder of one member.  The kernel keeps one per lane and advances all lanes of a warp in
// lock step (one symbol per step), so that lanes never drift apart into separately scheduled fragments;
// the host test simply calls the same steps in a loop.
struct Decoder {
    enum State { NEED_BLOCK = 0, SYMBOLS = 1, DONE = 2 };
    Bits br;
    int64_t opos, o0, o1, olim, dend;   // dend = c1 - 8: one past the deflate data
    int state, status;
    bool last;
    // segment mode: decoding starts at a zran checkpoint (a deflate block boundary in the middle of a stream) and ends
    // when the output reaches o1 -- the next checkpoint, also a block boundary -- or with the stream's last block
    bool seg;
    const uint8_t *win;
    int wlen;

    FXI_HD void fail(int code) { status = code; state = DONE; }

    // raw deflate data from compressed offset `cpos`; `bits` (0..7) leading bits of the block sit in the byte before it
    // (zran's convention: inflatePrime(bits, in[cpos - 1] >> (8 - bits))); `w` = the wl bytes of output before o0
    FXI_HD void begin_at(const uint8_t *in, int64_t in_size, int64_t cpos, int bits, int64_t out_cap, int64_t o0_, int64_t o1_,
                         const uint8_t *w, int wl) {
        status = INF_OK; state = NEED_BLOCK; last = false;
        seg = true; win = w; wlen = wl;
        o0 = o0_; o1 = o1_; opos = o0_; olim = o1_ < out_cap ? o1_ : out_cap; dend = in_size;
        br.in = in; br.pos = cpos; br.end = in_size; br.lim = in_size; br.buf = 0; br.nbits = 0;
        if (cpos < 0 || cpos > in_size || bits < 0 || bits > 7 || (bits && cpos < 1)) { fail(INF_BAD_HEADER); return; }
        if (bits) { br.buf = (uint64_t)(in[cpos - 1] >> (8 - bits)); br.nbits = bits; }
    }

    // gzip member header: 10 fixed bytes, FEXTRA (BGZF always), optional name/comment/crc
    FXI_HD void begin(const uint8_t *in, int64_t in_size, int64_t c0, int64_t c1, int64_t out_cap, int64_t o0_, int64_t o1_) {
        status = INF_OK; state = NEED_BLOCK; last = false;
        seg = false; win = nullptr; wlen = 0;
        o0 = o0_; o1 = o1_; opos = o0_; olim = o1_ < out_cap ? o1_ : out_cap; dend = c1 - 8;
        br.in = in; br.pos = c0; br.end = c1 - 8; br.lim = in_size; br.buf = 0; br.nbits = 0;
        int64_t p = c0;
        if (c1 - c0 < 18 + 8 || c1 > in_size || in[p] != 0x1f || in[p + 1] != 0x8b || in[p + 2] != 8) { fail(INF_BAD_HEADER); return; }
        const int flg = in[p + 3];
        p += 10;
        if (flg & 4) { const int xlen = in[p] | (in[p + 1] << 8); p += 2 + xlen; }
        if (flg & 8) { while (p < c1 && in[p]) ++p; ++p; }
        if (flg & 16) { while (p < c1 && in[p]) ++p; ++p; }
        if (flg & 2) p += 2;
        if (p > c1 - 8) { fail(INF_BAD_HEADER); return; }
        br.pos = p;
    }

    // A member's deflate data must end in the byte before its trailer: zlib reads the trailer right after the last
    // block, so bytes in between fail its CRC check even when the trailer describes the output correctly.
    FXI_HD void finish_member() {
        if (status == INF_OK && opos != o1) status = INF_SIZE;
        else if (status == INF_OK && !seg && br.pos - (br.nbits >> 3) != dend) status = INF_BAD_BLOCK;
        state = DONE;
    }

    // block header (+ stored data, + code lengths and tables): NEED_BLOCK -> SYMBOLS | NEED_BLOCK | DONE
    FXI_HD void begin_block(uint8_t *out, MemberTables &T, const DeflateConsts &K) {
        if (last || (seg && opos >= o1)) { finish_member(); return; }
        last = br.get(1) != 0;
        const int btype = (int)br.get(2);
        int hlit = 0, hdist = 0;
        uint8_t lens[320];                                   // code lengths of this block (thread-local)
        if (btype == 0) {
            br.drop(br.nbits & 7);                           // to a byte boundary
            const uint32_t len = br.get(16), nlen = br.get(16);
            if ((len ^ 0xffffu) != nlen) { fail(INF_BAD_BLOCK); return; }
            const int64_t src = br.pos - (br.nbits >> 3);
            if (src + (int64_t)len > dend || opos + (int64_t)len > olim) { fail(INF_OVERRUN); return; }
            for (uint32_t i = 0; i < len; ++i) out[opos + i] = br.in[src + i];
            opos += len;
            br.pos = src + len; br.buf = 0; br.nbits = 0;
            return;                                           // still NEED_BLOCK (or the end, next step)
        } else if (btype == 1) {
            for (int i = 0; i < 288; ++i) lens[i] = (uint8_t)(i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8)));
            for (int i = 0; i < 32; ++i) lens[288 + i] = 5;      // all 32 codes: a complete code; 30 and 31 are rejected when read
            hlit = 288; hdist = 32;
        } else if (btype == 2) {
            hlit = (int)br.get(5) + 257;
            hdist = (int)br.get(5) + 1;
            const int hclen = (int)br.get(4) + 4;
            if (hlit > 286 || hdist > 30) { fail(INF_BAD_BLOCK); return; }
            // code-length code: tiny canonical decoder, bit by bit
            uint8_t cl[19];
            for (int i = 0; i < 19; ++i) cl[i] = 0;
            int kraft = 0;                                   // code space the code-length code fills, of 128
            for (int i = 0; i < hclen; ++i) {
                const int v = (int)br.get(3);
                cl[K.CL_ORDER[i]] = (uint8_t)v;
                kraft += v ? 128 >> v : 0;
            }
            if (kraft != 128) { fail(INF_BAD_CODE); return; }   // complete, as zlib requires
            uint16_t ccnt[8], csym[19], offs[8];
            for (int i = 0; i < 8; ++i) ccnt[i] = 0;
            for (int i = 0; i < 19; ++i) ccnt[cl[i]]++;
            offs[1] = 0;
            for (int i = 1; i < 7; ++i) offs[i + 1] = (uint16_t)(offs[i] + ccnt[i]);
            for (int i = 0; i < 19; ++i)
                if (cl[i]) csym[offs[cl[i]]++] = (uint16_t)i;
            int idx = 0;
            while (idx < hlit + hdist) {
                int code = 0, first = 0, index = 0, sym = -1;
                for (int len = 1; len <= 7; ++len) {
                    code |= (int)br.get(1);
                    const int count = ccnt[len];
                    if (code - count < first) { sym = csym[index + (code - first)]; break; }
                    index += count; first += count; first <<= 1; code <<= 1;
                }
                if (sym < 0) { fail(INF_BAD_CODE); return; }
                if (sym < 16) lens[idx++] = (uint8_t)sym;
                else {
                    int rep, val = 0;
                    if (sym == 16) { if (idx == 0) { fail(INF_BAD_CODE); return; } val = lens[idx - 1]; rep = 3 + (int)br.get(2); }
                    else if (sym == 17) rep = 3 + (int)br.get(3);
                    else rep = 11 + (int)br.get(7);
                    if (idx + rep > hlit + hdist) { fail(INF_BAD_CODE); return; }
                    while (rep--) lens[idx++] = (uint8_t)val;
                }
            }
            if (lens[256] == 0) { fail(INF_BAD_CODE); return; }
        } else { fail(INF_BAD_BLOCK); return; }
        if (br.overrun()) { fail(INF_OVERRUN); return; }
        bool ok = build_table(lens, hlit, T.lit, TL_BITS, 9, T.litcnt, T.litsym);
        ok = build_table(lens + hlit, hdist, T.dist, TD_BITS, 5, T.distcnt, T.distsym) && ok;
        // over-subscribed or incomplete codes are invalid, except a single one-bit code and an empty distance code
        if (!ok) { fail(INF_BAD_CODE); return; }
        state = SYMBOLS;
    }

    // one literal, match or end-of-block
    FXI_HD void step_symbol(uint8_t *out, int64_t out_cap, const MemberTables &T, const DeflateConsts &K) {
        br.refill();
        int sym;
        const uint16_t e = T.lit[br.peek(TL_BITS)];
        if (e) { br.drop(e >> 9); sym = e & 511; }
        else sym = slow_decode(br, T.litcnt, T.litsym);
        if (sym < 0) { fail(INF_BAD_CODE); return; }
        if (sym < 256) {
            if (opos >= olim) { fail(INF_OVERRUN); return; }
            out[opos++] = (uint8_t)sym;
            return;
        }
        if (sym == 256) {
            if (br.overrun()) { fail(INF_OVERRUN); return; }
            state = NEED_BLOCK;
            return;
        }
        sym -= 257;
        if (sym >= 29) { fail(INF_BAD_CODE); return; }
        br.refill();
        const int mlen = K.LEN_BASE[sym] + (int)br.peek(K.LEN_EXTRA[sym]);
        br.drop(K.LEN_EXTRA[sym]);
        br.refill();
        int ds;
        const uint16_t de = T.dist[br.peek(TD_BITS)];
        if (de) { br.drop(de >> 5); ds = de & 31; }
        else ds = slow_decode(br, T.distcnt, T.distsym);
        if (ds < 0 || ds >= 30) { fail(INF_BAD_CODE); return; }
        br.refill();
        const int mdist = K.DIST_BASE[ds] + (int)br.peek(K.DIST_EXTRA[ds]);
        br.drop(K.DIST_EXTRA[ds]);
        if (mdist > opos - o0 + wlen) { fail(INF_BAD_CODE); return; }     // BGZF members are self-contained (wlen = 0)
        if (opos + mlen > olim) { fail(INF_OVERRUN); return; }
        copy_match(out, opos, opos - mdist, mlen, out_cap, o0, win, wlen);
        opos += mlen;
    }
};

// Decode the gzip member in[c0, c1) into out[o0, o1) start to finish (host test driver; the kernel
// interleaves the same steps across the lanes of a warp).  Returns an INF_* status.
FXI_HD int inflate_member(const uint8_t *in, int64_t in_size, int64_t c0, int64_t c1, uint8_t *out, int64_t out_cap,
                          int64_t o0, int64_t o1, MemberTables &T, const DeflateConsts &K) {
    Decoder d;
    d.begin(in, in_size, c0, c1, out_cap, o0, o1);
    while (d.state != Decoder::DONE) {
        if (d.state == Decoder::NEED_BLOCK) d.begin_block(out, T, K);
        else d.step_symbol(out, out_cap, T, K);
    }
    return d.status;
}

// Decode the deflate data from a zran checkpoint (cpos, bits, window) into out[o0, o1) start to finish.
FXI_HD int inflate_segment(const uint8_t *in, int64_t in_size, int64_t cpos, int bits, uint8_t *out, int64_t out_cap,
                           int64_t o0, int64_t o1, const uint8_t *win, int wlen, MemberTables &T, const DeflateConsts &K) {
    Decoder d;
    d.begin_at(in, in_size, cpos, bits, out_cap, o0, o1, win, wlen);
    while (d.state != Decoder::DONE) {
        if (d.state == Decoder::NEED_BLOCK) d.begin_block(out, T, K);
        else d.step_symbol(out, out_cap, T, K);
    }
    return d.status;
}

}  // namespace fxi
