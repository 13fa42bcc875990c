"""A byte-level baseline JPEG writer for decoder tests.

It takes quantised coefficient blocks (zig-zag order) and writes the marker segments and the Huffman-coded scan itself, so a
test controls what no real encoder lets it choose: the marker layout, the Huffman tables, where byte stuffing and restart
markers fall in the stream, and where the stream is cut.  There is no forward DCT and no attempt at any particular image.

`write_jpeg` returns a `Jpeg`: the bytes plus the byte offsets where each scan starts and where decoding resumes after each
RSTn, so that tests can assert the layout they meant to build."""
from __future__ import annotations

import heapq
from dataclasses import dataclass, field

import numpy as np

# natural (row-major) index of zig-zag position k
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# ITU T.81 Annex K.3 tables: (codes per length 1..16, symbols in code order)
_AC_TAIL = [0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a,
            0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77,
            0x78, 0x79, 0x7a]
STD_DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
STD_DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
STD_AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d],
               [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
                0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
                0x17, 0x18, 0x19, 0x1a] + _AC_TAIL + [0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
                0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
                0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
                0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
                0xf9, 0xfa])
STD_AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77],
                 [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
                  0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
                  0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a] + _AC_TAIL[13:] +
                 [0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3,
                  0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
                  0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7,
                  0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa])
AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]     # every baseline AC symbol


class Huff:
    """A Huffman table as DHT stores it (counts per code length, symbols in code order) and its canonical codes."""

    def __init__(self, bits, vals):
        self.bits, self.vals = [int(b) for b in bits], [int(v) for v in vals]
        assert len(self.bits) == 16 and sum(self.bits) == len(self.vals) <= 256
        self.code = {}
        c, k = 0, 0
        for ln in range(1, 17):
            for _ in range(self.bits[ln - 1]):
                self.code[self.vals[k]] = (c, ln); c += 1; k += 1
            assert c <= (1 << ln), "over-subscribed code lengths"
            c <<= 1

    def spec(self) -> bytes:
        return bytes(self.bits) + bytes(self.vals)


def std_tables():
    return {"dc": [Huff(*STD_DC_LUMA), Huff(*STD_DC_CHROMA)], "ac": [Huff(*STD_AC_LUMA), Huff(*STD_AC_CHROMA)]}


def crafted(lengths: dict) -> Huff:
    """Table with the given code length per symbol (canonical order: by length, then in the dict's order)."""
    order = sorted(lengths, key=lambda s: lengths[s])
    bits = [0] * 16
    for s in order: bits[lengths[s] - 1] += 1
    return Huff(bits, order)


def optimal(freq: dict) -> Huff:
    """Code lengths from symbol statistics, limited to 16 bits with the all-ones code left unused (T.81 Annex K.2)."""
    syms = [s for s in freq if freq[s] > 0]
    f = {s: freq[s] for s in syms}
    f[256] = 0                                        # reserved symbol: keeps every real code off the all-ones pattern
    heap = [(c, i, [s]) for i, (s, c) in enumerate(sorted(f.items()))]
    heapq.heapify(heap)
    size = {s: 0 for s in f}
    n = len(heap)
    while len(heap) > 1:
        c1, _, a = heapq.heappop(heap); c2, _, b = heapq.heappop(heap)
        for s in a + b: size[s] += 1
        heapq.heappush(heap, (c1 + c2, n, a + b)); n += 1
    bits = [0] * 33
    for s in f: bits[max(size[s], 1)] += 1
    for i in range(32, 16, -1):                       # Annex K.2 Adjust_BITS
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0: j -= 1
            bits[i] -= 2; bits[i - 1] += 1; bits[j + 1] += 2; bits[j] -= 1
    i = 16
    while bits[i] == 0: i -= 1
    bits[i] -= 1                                      # drop the reserved symbol (it has the longest code)
    order = sorted(syms, key=lambda s: (size[s], s))
    return Huff(bits[1:17], order)


@dataclass
class Comp:
    cid: int          # component id written in SOF / SOS
    h: int = 1
    v: int = 1
    tq: int = 0       # quantisation table id
    td: int = 0       # DC Huffman table id
    ta: int = 0       # AC Huffman table id


@dataclass
class Jpeg:
    data: bytes
    scan_starts: list = field(default_factory=list)     # first entropy-coded byte of each scan
    resumes: list = field(default_factory=list)         # first byte after each RSTn marker
    mcux: int = 0
    mcuy: int = 0


def geometry(W, H, comps):
    hmax = max(c.h for c in comps); vmax = max(c.v for c in comps)
    mcux = -(-W // (8 * hmax)); mcuy = -(-H // (8 * vmax))
    return hmax, vmax, mcux, mcuy


def block_grid(W, H, comps):
    """(rows, cols) of the padded block grid of each component: what `write_jpeg` expects in `blocks`"""
    _, _, mcux, mcuy = geometry(W, H, comps)
    return [(mcuy * c.v, mcux * c.h) for c in comps]


def category(v: int) -> int:
    return int(abs(int(v))).bit_length()


class BitWriter:
    def __init__(self):
        self.out = bytearray(); self.acc = 0; self.n = 0

    def put(self, code: int, length: int):
        self.acc = (self.acc << length) | (code & ((1 << length) - 1)); self.n += length
        while self.n >= 8:
            self.n -= 8
            b = (self.acc >> self.n) & 0xFF
            self.out.append(b)
            if b == 0xFF: self.out.append(0)                 # byte stuffing
        self.acc &= (1 << self.n) - 1

    def pad(self):                                     # 1-bits to the byte boundary; an all-ones byte is stuffed like any other
        if self.n: self.put((1 << (8 - self.n)) - 1, 8 - self.n)


def extra_bits(v: int, s: int) -> int:
    return v if v >= 0 else v + (1 << s) - 1


def encode_block(bw: BitWriter, blk, diff: int, dc: Huff, ac: Huff, zrl_tail=False):
    s = category(diff)
    bw.put(*dc.code[s])
    if s: bw.put(extra_bits(diff, s), s)
    last = max([k for k in range(1, 64) if blk[k] != 0], default=0)
    run = 0
    for k in range(1, last + 1):
        v = int(blk[k])
        if v == 0: run += 1; continue
        while run > 15: bw.put(*ac.code[0xF0]); run -= 16
        s = category(v)
        bw.put(*ac.code[(run << 4) | s]); bw.put(extra_bits(v, s), s); run = 0
    if last < 63:
        gap = 63 - last
        if zrl_tail and gap % 16 == 0:                 # ZRLs up to k = 64 exactly, no EOB
            for _ in range(gap // 16): bw.put(*ac.code[0xF0])
        else:
            bw.put(*ac.code[0x00])


def segment(marker: int, body: bytes, fill: int = 0) -> bytes:
    return b"\xff" * fill + bytes([0xFF, marker]) + (len(body) + 2).to_bytes(2, "big") + body


def write_jpeg(W, H, comps, blocks, quant, dc, ac, *, restart=0, dri="before_dht", tables_after_sof=False, one_dqt=False, one_dht=False,
               app=(), fill=0, rst_fill=0, sos_order=None, scans=None, redefine=False, sof=0xC0, dqt_precision=0, header_dc=None,
               header_ac=None, zrl_tail=False, eoi=True, eoi_fill=0) -> Jpeg:
    """comps: list of Comp; blocks[i]: int array (rows, cols, 64) in zig-zag order over the padded grid of `block_grid`;
    quant: {table id: 64 values in zig-zag order}; dc / ac: {table id: Huff}.
    restart: DRI interval (0 with dri != "none" writes DRI = 0); dri: "before_dht" | "after_dht" | "none";
    tables_after_sof: DQT / DHT after SOF; one_dqt / one_dht: all tables in one segment; app: extra APPn / COM segments as
    (marker, body); fill: 0xFF fill bytes before every marker segment; rst_fill / eoi_fill: fill bytes before every RSTn / the
    EOI (stb v2.08 takes a fill byte right after the scan for data and rejects the stream);
    sos_order: component order inside an interleaved scan; scans: list of component-index tuples, one per scan (default one
    interleaved scan); redefine: every table is first written with wrong contents and then again with the right ones;
    header_dc / header_ac: tables written to DHT instead of the ones the scan is coded with (damaged streams)."""
    ids = range(len(comps))
    out = bytearray(b"\xff\xd8")
    for m, body in app: out += segment(m, body, fill)

    def dqt():
        segs = []
        for t, q in sorted(quant.items()):
            q = [int(x) for x in q]
            body = bytes([(dqt_precision << 4) | t]) + (b"".join(x.to_bytes(2, "big") for x in q) if dqt_precision else bytes(q))
            segs.append(body)
        if redefine:
            segs = [bytes([s[0]]) + bytes(len(s) - 1) for s in segs] + segs      # all-zero tables first, then the real ones
        return segment(0xDB, b"".join(segs), fill) if one_dqt else b"".join(segment(0xDB, s, fill) for s in segs)

    def dht():
        hd, ha = header_dc or dc, header_ac or ac
        segs = [bytes([0x00 | t]) + h.spec() for t, h in sorted(hd.items())] + [bytes([0x10 | t]) + h.spec() for t, h in sorted(ha.items())]
        if redefine:
            segs = [bytes([s[0]]) + Huff([2] + [0] * 15, [0, 1]).spec() for s in segs] + segs
        return segment(0xC4, b"".join(segs), fill) if one_dht else b"".join(segment(0xC4, s, fill) for s in segs)

    dri_seg = b"" if dri == "none" else segment(0xDD, int(restart).to_bytes(2, "big"), fill)
    tables = dqt() + (dri_seg + dht() if dri == "before_dht" else dht() + dri_seg)
    sof_body = bytes([8]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([len(comps)])
    for c in comps: sof_body += bytes([c.cid, (c.h << 4) | c.v, c.tq])
    sof_seg = segment(sof, sof_body, fill)
    out += (sof_seg + tables) if tables_after_sof else (tables + sof_seg)

    hmax, vmax, mcux, mcuy = geometry(W, H, comps)
    res = Jpeg(b"", mcux=mcux, mcuy=mcuy)
    for scan in (scans or [tuple(sos_order or ids)]):
        sos = bytes([len(scan)]) + b"".join(bytes([comps[i].cid, (comps[i].td << 4) | comps[i].ta]) for i in scan) + bytes([0, 63, 0])
        out += segment(0xDA, sos, fill)
        res.scan_starts.append(len(out))
        if len(scan) == 1:                             # non-interleaved: one block per MCU over the component's own extent
            c = comps[scan[0]]
            bw_, bh_ = -(-(-(-W * c.h // hmax)) // 8), -(-(-(-H * c.v // vmax)) // 8)
            units = [[(scan[0], by, bx)] for by in range(bh_) for bx in range(bw_)]
        else:
            units = [[(i, my * comps[i].v + y, mx * comps[i].h + x) for i in scan for y in range(comps[i].v) for x in range(comps[i].h)]
                     for my in range(mcuy) for mx in range(mcux)]
        bw = BitWriter(); pred = {i: 0 for i in ids}; rst = 0
        for u, unit in enumerate(units):
            if restart and u and u % restart == 0:
                bw.pad(); out += bw.out; bw = BitWriter()
                out += b"\xff" * rst_fill + bytes([0xFF, 0xD0 + (rst & 7)]); rst += 1
                res.resumes.append(len(out)); pred = {i: 0 for i in ids}
            for i, by, bx in unit:
                blk = blocks[i][by, bx]
                c = comps[i]
                encode_block(bw, blk, int(blk[0]) - pred[i], dc[c.td], ac[c.ta], zrl_tail)
                pred[i] = int(blk[0])
        bw.pad(); out += bw.out
    if eoi: out += b"\xff" * eoi_fill + b"\xff\xd9"
    res.data = bytes(out)
    return res


def stats(comps, blocks, restart=0, zrl_tail=False):
    """Symbol counts per (kind, table id) of one interleaved scan: the input of `optimal`"""
    cnt = {}
    class Counter:                                      # stands in for a Huff: counts every symbol it is asked to code
        def __init__(self, key): self.key = key
        @property
        def code(self): return self
        def __getitem__(self, s): cnt.setdefault(self.key, {}); cnt[self.key][s] = cnt[self.key].get(s, 0) + 1; return (0, 1)
    H = blocks[0].shape[0] * 8; W = blocks[0].shape[1] * 8          # (comps[0] is the full-resolution component)
    std = std_tables()
    write_jpeg(W, H, comps, blocks, {c.tq: [1] * 64 for c in comps}, {c.td: Counter(("dc", c.td)) for c in comps},
               {c.ta: Counter(("ac", c.ta)) for c in comps}, restart=restart, zrl_tail=zrl_tail,
               header_dc={c.td: std["dc"][0] for c in comps}, header_ac={c.ta: std["ac"][0] for c in comps})
    return cnt


def random_blocks(rng, grid, *, dc_range=300, ac_max=40, density=0.25, q=None):
    """Blocks of random coefficients: DC in [-dc_range, dc_range], a fraction `density` of the AC terms non-zero, decaying
    with frequency, and a zero block here and there."""
    out = []
    for rows, cols in grid:
        b = np.zeros((rows, cols, 64), np.int32)
        b[..., 0] = rng.integers(-dc_range, dc_range + 1, (rows, cols))
        k = np.arange(1, 64)
        amp = np.maximum(1, (ac_max / (1 + k / 6.0)).astype(np.int64))
        mask = rng.random((rows, cols, 63)) < density * np.exp(-k / 40.0)
        b[..., 1:] = np.where(mask, rng.integers(-amp, amp + 1, (rows, cols, 63)), 0)
        b[rng.random((rows, cols)) < 0.05, 1:] = 0
        out.append(b)
    return out


def ff_block(dc: Huff, ac: Huff, t: int):
    """A block (64 zig-zag coefficients, its DC taken as the difference from a zero predictor) whose coded bits, written from
    a byte boundary, make raw byte `t` 0xFF - so a stuffed `FF 00` pair starts at byte t counted from the scan start or from
    the RSTn the block follows.  Found by search over padding coefficients of sizes 7, 1 and 2 followed by a run of ones
    (a size-10 coefficient of value 1023), or, for t = 0, by a large DC difference."""
    def raw(blk):
        bw = BitWriter(); encode_block(bw, blk, int(blk[0]), dc, ac); return bytes(bw.out)
    cands = []
    for dcv in (0, 1024 + 512, -1):
        cands.append((dcv, 0, 0, 0))
        for n7 in range(18):
            for a in range(8):
                for b in range(3):
                    cands.append((dcv, n7, a, b))
    for dcv, n7, a, b in cands:
        if n7 + a + b + 1 > 63: continue
        blk = np.zeros(64, np.int32); blk[0] = dcv
        k = 1
        for _ in range(n7): blk[k] = 64; k += 1
        for _ in range(a): blk[k] = -1; k += 1
        for _ in range(b): blk[k] = 2; k += 1
        blk[k] = 1023
        r = raw(blk)
        if len(r) > t + 1 and r[t] == 0xFF and r[t + 1] == 0 and 0xFF not in r[:t]:
            return blk
    raise ValueError(f"no block puts FF at byte {t}")


def grey(n=1):
    return [Comp(1 + i, 1, 1, 0, 0, 0) for i in range(n)]


def ycc(h, v, cid0=1, luma_tabs=(0, 0, 0), chroma_tabs=(1, 1, 1)):
    """Y at (h, v), Cb and Cr at 1x1, with (tq, td, ta) per luma / chroma"""
    return [Comp(cid0, h, v, *luma_tabs), Comp(cid0 + 1, 1, 1, *chroma_tabs), Comp(cid0 + 2, 1, 1, *chroma_tabs)]


def std_quant(scale=1):
    """two plausible quantisation tables (zig-zag order), multiplied by `scale` and clipped to 1..255"""
    k = np.arange(64)
    return {0: np.clip((2 + k // 3) * scale, 1, 255).astype(int), 1: np.clip((3 + k // 2) * scale, 1, 255).astype(int)}
