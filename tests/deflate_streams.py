"""A raw deflate bit writer for decoder tests (RFC 1950 / 1951).

The caller chooses everything zlib chooses for itself: the token list (literals and length/distance pairs), where blocks
start and end, each block's type, and for dynamic blocks the code lengths, HLIT / HDIST / HCLEN and the run-length coding
of the code lengths.  `zlib_stream` adds the zlib header and the Adler-32 trailer."""
from __future__ import annotations

import zlib

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
             12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def len_code(n):
    i = max(i for i in range(29) if LEN_BASE[i] <= n)
    return 257 + i, LEN_EXTRA[i], n - LEN_BASE[i]


def dist_code(d):
    i = max(i for i in range(30) if DIST_BASE[i] <= d)
    return i, DIST_EXTRA[i], d - DIST_BASE[i]


def canonical(lengths):
    """symbol -> (code, length) for the canonical code of RFC 1951 3.2.2 (zero length = no code)"""
    mx = max(lengths, default=0)
    bl = [0] * (mx + 2)
    for ln in lengths:
        if ln: bl[ln] += 1
    code, nxt = 0, [0] * (mx + 2)
    for b in range(1, mx + 1):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = {}
    for s, ln in enumerate(lengths):
        if ln: out[s] = (nxt[ln], ln); nxt[ln] += 1
    return out


class Bits:
    """LSB-first bit writer; Huffman codes are written most significant bit first"""

    def __init__(self):
        self.out = bytearray(); self.acc = 0; self.n = 0

    def put(self, v, n):
        self.acc |= (v & ((1 << n) - 1)) << self.n; self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 0xFF); self.acc >>= 8; self.n -= 8

    def code(self, c, n):
        self.put(int(format(c, f"0{n}b")[::-1], 2), n)

    def align(self):
        if self.n: self.put(0, 8 - self.n)

    def bytes(self):
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def decode_tokens(tokens) -> bytes:
    """The bytes a token list stands for (literal: int 0-255; match: (length, distance))."""
    out = bytearray()
    for t in tokens:
        if isinstance(t, int): out.append(t)
        else:
            ln, d = t
            for _ in range(ln): out.append(out[-d])
    return bytes(out)


def huffman_lengths(freq: dict, nsym: int, max_len: int) -> list:
    """Code lengths of a Huffman code for the symbols with a non-zero count; a balanced complete code instead when that
    one would be longer than max_len.  A single used symbol gets a partner so that the code is complete."""
    import heapq
    syms = [s for s in sorted(freq) if freq[s]]
    if len(syms) == 1: syms.append((syms[0] + 1) % nsym)
    lens = [0] * nsym
    heap = [(freq.get(s, 0), i, [s]) for i, s in enumerate(syms)]
    heapq.heapify(heap); k = len(heap)
    while len(heap) > 1:
        c1, _, a = heapq.heappop(heap); c2, _, b = heapq.heappop(heap)
        for s in a + b: lens[s] += 1
        heapq.heappush(heap, (c1 + c2, k, a + b)); k += 1
    if max(lens) > max_len:
        depth = (len(syms) - 1).bit_length()
        short = (1 << depth) - len(syms)                # this many symbols fit one level up
        ranked = sorted(syms, key=lambda s: -freq.get(s, 0))
        lens = [0] * nsym
        for i, s in enumerate(ranked): lens[s] = depth - 1 if i < short else depth
    return lens


def lengths_from_tokens(tokens):
    """literal/length and distance code lengths for the symbols a token list uses, plus end-of-block"""
    lf, df = {256: 1}, {}
    for t in tokens:
        if isinstance(t, int): lf[t] = lf.get(t, 0) + 1
        else:
            s, _, _ = len_code(t[0]); lf[s] = lf.get(s, 0) + 1
            d, _, _ = dist_code(t[1]); df[d] = df.get(d, 0) + 1
    return huffman_lengths(lf, 286, 15), (huffman_lengths(df, 30, 15) if df else [1] + [0] * 29)


def rle_lengths(lens):
    """code-length symbols (sym, extra bits, extra value) for a list of lengths, with repeat codes 16 / 17 / 18 where they fit"""
    out, i = [], 0
    while i < len(lens):
        v = lens[i]; run = 1
        while i + run < len(lens) and lens[i + run] == v: run += 1
        if v == 0 and run >= 11:
            r = min(run, 138); out.append((18, 7, r - 11)); i += r; continue
        if v == 0 and run >= 3:
            r = min(run, 10); out.append((17, 3, r - 3)); i += r; continue
        out.append((v, 0, 0)); i += 1
        run -= 1
        while run >= 3:
            r = min(run, 6); out.append((16, 2, r - 3)); i += r; run -= r
    return out


class Deflate:
    """Raw deflate writer: blocks are appended one at a time; `bits` is the shared bit stream."""

    def __init__(self):
        self.bits = Bits()

    def stored(self, data: bytes, last=False, nlen=None):
        b = self.bits
        b.put(int(last), 1); b.put(0, 2); b.align()
        b.put(len(data), 16); b.put((~len(data) & 0xFFFF) if nlen is None else nlen, 16)
        for x in data: b.put(x, 8)

    def _tokens(self, tokens, lit, dist):
        b = self.bits
        for t in tokens:
            if isinstance(t, int): b.code(*lit[t])
            else:
                ln, d = t
                s, ne, ev = len_code(ln); b.code(*lit[s]); b.put(ev, ne)
                s, ne, ev = dist_code(d); b.code(*dist[s]); b.put(ev, ne)
        if 256 in lit: b.code(*lit[256])                 # (a code without end-of-block is a malformed stream on purpose)

    def fixed(self, tokens, last=False):
        self.bits.put(int(last), 1); self.bits.put(1, 2)
        self._tokens(tokens, canonical(FIXED_LIT), canonical(FIXED_DIST))

    def dynamic(self, tokens, last=False, lit_lens=None, dist_lens=None, hlit=None, hdist=None, cl_syms=None, cl_lens=None, hclen=None):
        """lit_lens / dist_lens: code lengths (default: a Huffman code of the tokens); hlit / hdist: how many of them to send
        (default: up to the last non-zero one); cl_syms: the code-length symbols as (sym, extra bits, value), default
        `rle_lengths` over the sent lengths; cl_lens: code lengths of the code-length code (default: a Huffman code of cl_syms)."""
        if lit_lens is None or dist_lens is None:
            ll, dl = lengths_from_tokens(tokens)
            lit_lens = ll if lit_lens is None else lit_lens
            dist_lens = dl if dist_lens is None else dist_lens
        lit_lens = list(lit_lens) + [0] * (286 - len(lit_lens)); dist_lens = list(dist_lens) + [0] * (30 - len(dist_lens))
        if hlit is None: hlit = max(257, max(i for i, x in enumerate(lit_lens) if x) + 1)
        if hdist is None: hdist = max(1, max((i for i, x in enumerate(dist_lens) if x), default=0) + 1)
        sent = lit_lens[:hlit] + dist_lens[:hdist]
        if cl_syms is None: cl_syms = rle_lengths(sent)
        if cl_lens is None:
            freq = {}
            for s, _, _ in cl_syms: freq[s] = freq.get(s, 0) + 1
            cl_lens = huffman_lengths(freq, 19, 7)
        if hclen is None: hclen = max(4, max(i for i, s in enumerate(CL_ORDER) if cl_lens[s]) + 1)
        b = self.bits
        b.put(int(last), 1); b.put(2, 2)
        b.put(hlit - 257, 5); b.put(hdist - 1, 5); b.put(hclen - 4, 4)
        for i in range(hclen): b.put(cl_lens[CL_ORDER[i]], 3)
        clc = canonical(cl_lens)
        for s, ne, ev in cl_syms:
            b.code(*clc[s])
            if ne: b.put(ev, ne)
        self._tokens(tokens, canonical(lit_lens), canonical(dist_lens))

    def raw(self) -> bytes:
        return self.bits.bytes()


def zlib_stream(raw_deflate: bytes, data: bytes) -> bytes:
    return b"\x78\x01" + raw_deflate + zlib.adler32(data).to_bytes(4, "big")
