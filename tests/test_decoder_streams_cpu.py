"""CPU: hand-built JPEG and deflate streams (tests/jpeg_streams.py, tests/deflate_streams.py) through the host decoders.

JPEG: every valid crafted stream must be accepted by the compiled reference (stb_image v2.08 through ml::SensorData,
oracle/_ref/libref_sens.so) and the host decoder (jpeg.cpp) must give its bytes.  The streams vary what libjpeg never
does: marker layout, Huffman tables (optimal, every AC code 16 bits long, codes at exactly 9 and 10 bits), where `FF 00`
stuffing and RSTn markers fall, coefficient extremes.  Deflate: every crafted stream must equal zlib.decompress and the host
build of the GPU inflate (inflate.cu).

The stream families are functions so that test_decoder_streams_gpu.py decodes the same bytes on the device."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest

import deflate_streams as ds
import jpeg_streams as js
from scannet_b200 import ScnError, sens, synth
from scannet_b200.sens import SensFile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref_sens.so")
need_ref = pytest.mark.skipif(not os.path.exists(REF_SO), reason="oracle/_ref not built (needs the reference sources)")


# ---- decoding through a .sens container ---------------------------------------------------------------------------------------
def write_container(path, jpegs, W, H):
    n = len(jpegs)
    it = iter(jpegs)
    synth.write_sens(str(path), np.full((n, 8, 8), 1000, np.uint16), np.zeros((n, 1, 1, 3), np.uint8), np.tile(np.eye(4, dtype=np.float32), (n, 1, 1)),
                     np.eye(4, dtype=np.float32), depth_comp=0, color_comp=2, jpeg_encoder=lambda x: next(it))
    # the colour size in the header is the frame size the decoders check against
    with open(path, "r+b") as f:
        data = f.read()
        off = 4 + 8 + len(b"synthetic") + 4 * 64 + 8
        f.seek(off); f.write(int(W).to_bytes(4, "little") + int(H).to_bytes(4, "little"))
    return str(path)


def host_colors(path, n):
    """the library's host decoder: an RGB8 array per frame, or the ScnError it raised"""
    s = SensFile(path); out = []
    for i in range(n):
        try: out.append(s.color(i))
        except ScnError as e: out.append(e)
    return s, out


def ref_colors(path, n, W, H):
    """stb_image through the unmodified reference: an RGB8 array per frame, or None where it fails; None overall without it"""
    if not os.path.exists(REF_SO): return None
    L = C.CDLL(REF_SO); L.ref_sens_open.restype = C.c_void_p; L.ref_sens_open.argtypes = [C.c_char_p]
    L.ref_sens_color.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]; L.ref_sens_close.argtypes = [C.c_void_p]
    r = L.ref_sens_open(path.encode()); assert r
    out = []
    for i in range(n):
        rc = np.zeros((H, W, 3), np.uint8)
        out.append(rc if L.ref_sens_color(r, i, rc.ctypes.data) == 0 else None)
    L.ref_sens_close(r)
    return out


def assert_host_matches_stb(tmp_path, name, jpegs, W, H):
    """every stream decodes on the host; where the reference is built, stb accepts it and gives the same bytes"""
    p = write_container(tmp_path / f"{name}.sens", jpegs, W, H)
    _, host = host_colors(p, len(jpegs))
    for i, h in enumerate(host):
        assert not isinstance(h, Exception), (name, i, h)
    ref = ref_colors(p, len(jpegs), W, H)
    if ref is not None:
        for i, (h, r) in enumerate(zip(host, ref)):
            assert r is not None, f"{name}[{i}]: stb rejects the stream"
            assert (h == r).all(), f"{name}[{i}]: host decoder differs from stb"
    return host


# ---- JPEG stream families -----------------------------------------------------------------------------------------------------
SAMPLINGS = {"444": (1, 1), "422": (2, 1), "420": (2, 2), "440": (1, 2), "grey": None}


def comps_for(sampling, cid0=1, swapped=False):
    if sampling == "grey": return [js.Comp(cid0, 1, 1, 2 if swapped else 0, 1 if swapped else 0, 1 if swapped else 0)]
    h, v = SAMPLINGS[sampling]
    if swapped: return js.ycc(h, v, cid0, luma_tabs=(2, 1, 1), chroma_tabs=(3, 0, 0))
    return js.ycc(h, v, cid0)


def table_kind(kind, comps, blocks, restart=0, zrl_tail=False):
    """(dc, ac) table dicts for the table ids the components use"""
    tds = sorted({c.td for c in comps}); tas = sorted({c.ta for c in comps})
    if kind == "std":
        t = js.std_tables()
        # luma tables on the luma component's ids, chroma tables on the others
        return ({d: t["dc"][0 if d == comps[0].td else 1] for d in tds}, {a: t["ac"][0 if a == comps[0].ta else 1] for a in tas})
    if kind == "optimal":
        st = js.stats(comps, blocks, restart=restart, zrl_tail=zrl_tail)
        return ({d: js.optimal(st[("dc", d)]) for d in tds}, {a: js.optimal(st[("ac", a)]) for a in tas})
    if kind == "long16":          # one DC symbol; every AC symbol 16 bits long: every AC code takes the slow path
        return ({d: js.crafted({0: 1}) for d in tds}, {a: js.crafted({s: 16 for s in js.AC_SYMBOLS}) for a in tas})
    if kind == "fast9_10":        # frequent symbols at exactly kFastBits = 9 bits, the rest at 10
        dc = js.crafted({s: (9 if s < 7 else 10) for s in range(12)})
        ac = js.crafted({s: (9 if (s & 15) <= 3 else 10) for s in js.AC_SYMBOLS})
        return ({d: dc for d in tds}, {a: ac for a in tas})
    raise ValueError(kind)


def content(rng, W, H, comps, kind):
    blocks = js.random_blocks(rng, js.block_grid(W, H, comps))
    if kind == "long16":
        for b in blocks: b[..., 0] = 0                                  # the one-symbol DC table codes difference 0 only
    return blocks


LAYOUTS = {
    "plain": {},
    "one_segment_tables": dict(one_dqt=True, one_dht=True),
    "tables_after_sof_dri0": dict(tables_after_sof=True, dri="after_dht", restart=0),
    "app_exif_com_fill": dict(app=[(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"), (0xE1, b"Exif\x00\x00" + bytes(range(256)) * 40),
                                   (0xFE, b"crafted")], fill=3),
    "redefined_tables_zero_ids": dict(redefine=True),
    "swapped_table_ids": dict(),
    "restart2_dri_before_dht": dict(restart=2, dri="before_dht"),
    "restart3_dri_after_dht": dict(restart=3, dri="after_dht"),
}


def layout_streams(sampling, kind, W=41, H=27, seed=0):
    """one stream per layout for a sampling and a table kind"""
    out = []
    for li, (name, opts) in enumerate(LAYOUTS.items()):
        rng = np.random.default_rng(1000 * seed + li)
        comps = comps_for(sampling, cid0=0 if name == "redefined_tables_zero_ids" else 1, swapped=name == "swapped_table_ids")
        blocks = content(rng, W, H, comps, kind)
        dc, ac = table_kind(kind, comps, blocks, restart=opts.get("restart", 0))
        q = js.std_quant(1 + li % 3)
        quant = {c.tq: q[c.tq & 1] for c in comps}
        out.append((f"{sampling}-{kind}-{name}", js.write_jpeg(W, H, comps, blocks, quant, dc, ac, **opts).data))
    return out


def coefficient_streams(sampling):
    """DC categories 0-11, AC sizes 1-10 (incl. +-1023 at q = 255: de-quantisation truncated to int16), zero runs of 15,
    ZRL chains ending at k = 64, a last coefficient at k = 63, all-zero blocks, and blocks past both IDCT clamp limits"""
    W, H = 48, 32
    comps = comps_for(sampling)
    grid = js.block_grid(W, H, comps)
    rng = np.random.default_rng(7)
    out = []
    # DC: alternate v and 0 so the differences cover every category with both signs and both ends of each category
    vals = [0] + [s * m for c in range(1, 12) for m in (1 << (c - 1), (1 << c) - 1) for s in (1, -1)]
    blocks = [np.zeros((r, c, 64), np.int32) for r, c in grid]
    seq = [v for x in vals for v in (x, 0)]
    for b in blocks:
        flat = b.reshape(-1, 64)
        flat[:, 0] = [seq[i % len(seq)] for i in range(len(flat))]
    q1 = {c.tq: np.ones(64, int) for c in comps}
    dc, ac = table_kind("std", comps, blocks)
    out.append(("dc-categories", js.write_jpeg(W, H, comps, blocks, q1, dc, ac).data))
    # AC sizes 1..10, one coefficient per block at a random position, q = 255 everywhere (1023 * 255 wraps in int16)
    blocks = [np.zeros((r, c, 64), np.int32) for r, c in grid]
    sizes = [(s, v) for s in range(1, 11) for v in ((1 << s) - 1, -((1 << s) - 1), 1 << (s - 1), -(1 << (s - 1)))]
    i = 0
    for b in blocks:
        for blk in b.reshape(-1, 64):
            s, v = sizes[i % len(sizes)]; i += 1
            blk[int(rng.integers(1, 64))] = v
    q255 = {c.tq: np.full(64, 255) for c in comps}
    out.append(("ac-sizes-q255", js.write_jpeg(W, H, comps, blocks, q255, dc, ac).data))
    # zero runs, ZRL chains to k = 64, k = 63, all-zero blocks
    blocks = [np.zeros((r, c, 64), np.int32) for r, c in grid]
    pats = [lambda b: b.__setitem__(16, 5),                           # run of 15 then a coefficient
            lambda b: (b.__setitem__(1, 3), b.__setitem__(17, -2)),   # run of 15 after k = 1
            lambda b: b.__setitem__(15, 7),                           # last at k = 15: 48 zeros -> ZRL x 3 ends at 64
            lambda b: b.__setitem__(47, -9),                          # last at k = 47: one ZRL to 64
            lambda b: b.__setitem__(63, 4),                           # last coefficient at k = 63, no EOB
            lambda b: (b.__setitem__(1, 1), b.__setitem__(34, 1), b.__setitem__(63, -1)),   # ZRL + run, then k = 63
            lambda b: None]                                           # all-zero block
    i = 0
    for b in blocks:
        for blk in b.reshape(-1, 64):
            pats[i % len(pats)](blk); blk[0] = (i % 5) * 20 - 40; i += 1
    q = js.std_quant(1)
    quant = {c.tq: q[c.tq & 1] for c in comps}
    out.append(("runs-zrl-k63", js.write_jpeg(W, H, comps, blocks, quant, dc, ac, zrl_tail=True).data))
    # IDCT clamps: huge DC either way, and a strong first AC term swinging a block past 0 and 255 at once
    blocks = [np.zeros((r, c, 64), np.int32) for r, c in grid]
    i = 0
    for b in blocks:
        for blk in b.reshape(-1, 64):
            kind = i % 4; i += 1
            if kind == 0: blk[0] = 1000
            elif kind == 1: blk[0] = -1000
            elif kind == 2: blk[1] = 250; blk[2] = -250
            else: blk[0] = 500; blk[1] = -300; blk[9] = 120
    q4 = {c.tq: np.full(64, 4) for c in comps}
    out.append(("idct-clamps", js.write_jpeg(W, H, comps, blocks, q4, dc, ac).data))
    return out


def stuffing_streams(sampling, restart=2):
    """`FF 00` at raw offsets 0..31 from the scan start and from every RSTn (offset 31 puts FF in the last byte of a 32-byte
    staging step of the device reader and the stuffed 00 in the first byte of the next).  Returns (name, Jpeg, t)."""
    W, H = 64, 48
    comps = comps_for(sampling)
    t_std = js.std_tables()
    out = []
    for t in range(32):
        rng = np.random.default_rng(100 + t)
        blocks = js.random_blocks(rng, js.block_grid(W, H, comps), dc_range=200)
        dc, ac = table_kind("std", comps, blocks)
        ffb = js.ff_block(dc[comps[0].td], ac[comps[0].ta], t)
        _, _, mcux, mcuy = js.geometry(W, H, comps)
        c0 = comps[0]
        for u in range(0, mcux * mcuy, restart):
            my, mx = divmod(u, mcux)
            blocks[0][my * c0.v, mx * c0.h] = ffb
        q = js.std_quant(1)
        j = js.write_jpeg(W, H, comps, blocks, {c.tq: q[c.tq & 1] for c in comps}, dc, ac, restart=restart)
        out.append((f"stuff-{sampling}-{t}", j, t))
    return out


def restart_streams(sampling, W, H, seed=3):
    """restart intervals 1, 2, mcux-1, mcux, mcux+1 and more than the MCU count; interval 1 wraps RST0..7 many times"""
    comps = comps_for(sampling)
    _, _, mcux, mcuy = js.geometry(W, H, comps)
    out = []
    for r in sorted({1, 2, max(1, mcux - 1), mcux, mcux + 1, mcux * mcuy + 5}):
        rng = np.random.default_rng(seed + r)
        blocks = js.random_blocks(rng, js.block_grid(W, H, comps))
        dc, ac = table_kind("std", comps, blocks)
        q = js.std_quant(2)
        out.append((f"rst{r}", js.write_jpeg(W, H, comps, blocks, {c.tq: q[c.tq & 1] for c in comps}, dc, ac, restart=r).data))
    return out


def simple_stream(W, H, sampling="420", seed=0, kind="std", **opts):
    comps = opts.pop("comps", None) or comps_for(sampling)
    rng = np.random.default_rng(seed)
    blocks = content(rng, W, H, comps, kind)
    dc, ac = table_kind(kind, comps, blocks, restart=opts.get("restart", 0))
    q = js.std_quant(1 + seed % 3)
    return js.write_jpeg(W, H, comps, blocks, {c.tq: q[c.tq & 1] for c in comps}, dc, ac, **opts)


def declined_streams(W=48, H=32):
    """valid streams the device path hands to the host decoder (16-bit DQT is an error everywhere: not in this list)"""
    out = [("411", simple_stream(W, H, comps=[js.Comp(1, 4, 1, 0, 0, 0), js.Comp(2, 1, 1, 1, 1, 1), js.Comp(3, 1, 1, 1, 1, 1)]).data)]
    t = js.std_tables()
    comps = [js.Comp(1, 2, 2, 0, 2, 0), js.Comp(2, 1, 1, 1, 1, 1), js.Comp(3, 1, 1, 1, 1, 1)]    # luma DC on Huffman table 2
    blocks = js.random_blocks(np.random.default_rng(5), js.block_grid(W, H, comps))
    q = js.std_quant(1)
    out.append(("huffman-id-2", js.write_jpeg(W, H, comps, blocks, {0: q[0], 1: q[1]}, {1: t["dc"][1], 2: t["dc"][0]}, {0: t["ac"][0], 1: t["ac"][1]}).data))
    out.append(("sos-order", simple_stream(W, H, seed=6, sos_order=[0, 2, 1]).data))
    out.append(("three-scans", simple_stream(W, H, seed=7, scans=[(0,), (1,), (2,)]).data))
    return out


def dqt16_stream(W=48, H=32):
    return simple_stream(W, H, seed=8, dqt_precision=1).data


def truncations(j: js.Jpeg, tail=64):
    """the scan cut at each of its last `tail` bytes: bare, followed by EOI, and followed by RST0 + EOI"""
    end = len(j.data) - 2                                               # the scan ends where EOI starts
    out = []
    for cut in range(end - tail, end):
        body = j.data[:cut]
        out += [(f"cut{cut}", body), (f"cut{cut}+eoi", body + b"\xff\xd9"), (f"cut{cut}+rst+eoi", body + b"\xff\xd0\xff\xd9")]
    return out


# ---- tests: JPEG ----------------------------------------------------------------------------------------------------------------
def test_standard_tables_are_libjpegs():
    """the Annex K tables of the writer are the ones libjpeg writes"""
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(0).integers(0, 255, (16, 16, 3)).astype(np.uint8)
    b = cv2.imencode(".jpg", img)[1].tobytes()
    want = {0x00: js.STD_DC_LUMA, 0x10: js.STD_AC_LUMA, 0x01: js.STD_DC_CHROMA, 0x11: js.STD_AC_CHROMA}
    i, seen = 2, 0
    while b[i + 1] != 0xDA:
        L = int.from_bytes(b[i + 2:i + 4], "big")
        if b[i + 1] == 0xC4:
            s = b[i + 4:i + 2 + L]
            while s:
                n = sum(s[1:17])
                assert (list(s[1:17]), list(s[17:17 + n])) == tuple(map(list, want[s[0]])); seen += 1
                s = s[17 + n:]
        i += 2 + L
    assert seen == 4


def test_writer_tables_and_stuffing_helper():
    """optimal tables are valid length-limited codes; ff_block puts FF 00 where it says"""
    rng = np.random.default_rng(0)
    for _ in range(20):
        freq = {s: int(rng.integers(0, 10 ** int(rng.integers(1, 7)))) for s in js.AC_SYMBOLS}
        h = js.optimal(freq)
        assert max(ln for _, ln in h.code.values()) <= 16
        assert sum(2.0 ** -ln for _, ln in h.code.values()) < 1.0                # the all-ones code stays free
        assert set(h.code) == {s for s in freq if freq[s]}
    t = js.std_tables()
    for tt in range(32):
        blk = js.ff_block(t["dc"][0], t["ac"][0], tt)
        bw = js.BitWriter(); js.encode_block(bw, blk, int(blk[0]), t["dc"][0], t["ac"][0])
        assert bw.out[tt] == 0xFF and bw.out[tt + 1] == 0


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
@pytest.mark.parametrize("kind", ["std", "optimal", "long16", "fast9_10"])
@need_ref
def test_layouts_and_tables_match_stb(tmp_path, built, sampling, kind):
    streams = layout_streams(sampling, kind)
    assert_host_matches_stb(tmp_path, f"{sampling}-{kind}", [s for _, s in streams], 41, 27)


@pytest.mark.parametrize("sampling", list(SAMPLINGS))
@need_ref
def test_coefficient_edges_match_stb(tmp_path, built, sampling):
    streams = coefficient_streams(sampling)
    assert_host_matches_stb(tmp_path, sampling, [s for _, s in streams], 48, 32)


@pytest.mark.parametrize("sampling", ["420", "grey"])
@need_ref
def test_stuffing_at_every_offset_matches_stb(tmp_path, built, sampling):
    streams = stuffing_streams(sampling)
    for name, j, t in streams:
        for r in j.scan_starts + j.resumes:
            assert j.data[r + t] == 0xFF and j.data[r + t + 1] == 0, (name, r)
    assert_host_matches_stb(tmp_path, sampling, [j.data for _, j, _ in streams], 64, 48)


@pytest.mark.parametrize("sampling,W,H", [("420", 40, 24), ("444", 24, 16), ("grey", 40, 8)])
@need_ref
def test_restart_intervals_match_stb(tmp_path, built, sampling, W, H):
    streams = restart_streams(sampling, W, H)
    assert_host_matches_stb(tmp_path, sampling, [s for _, s in streams], W, H)


@pytest.mark.parametrize("wh", [(1, 1), (1, 37), (37, 1), (497, 17), (33, 19)])
@pytest.mark.parametrize("sampling", ["420", "422", "440", "grey"])
@need_ref
def test_odd_sizes_match_stb(tmp_path, built, wh, sampling):
    W, H = wh
    assert_host_matches_stb(tmp_path, f"{sampling}-{W}x{H}", [simple_stream(W, H, sampling, seed=W + H).data], W, H)


@need_ref
def test_declined_streams_match_stb(tmp_path, built):
    streams = declined_streams()
    assert_host_matches_stb(tmp_path, "declined", [s for _, s in streams], 48, 32)
    p = write_container(tmp_path / "dqt16.sens", [dqt16_stream()], 48, 32)
    _, host = host_colors(p, 1)
    assert isinstance(host[0], ScnError)
    assert ref_colors(p, 1, 48, 32)[0] is None                      # stb v2.08 rejects 16-bit tables too


def truncation_cases():
    """(sampling, W, H, Jpeg, cases): scans without restart markers and with an interval of 5 MCUs, cut at each of their
    last 64 bytes (see `truncations`)"""
    out = []
    for seed, (sampling, restart) in enumerate([("420", 0), ("grey", 0), ("444", 0), ("420", 5), ("grey", 5)]):
        j = simple_stream(64, 48, sampling, seed=seed, restart=restart)
        out.append((sampling, 64, 48, j, truncations(j)))
    return out


@need_ref
def test_truncated_scans_against_stb(tmp_path, built):
    """A scan cut at each of its last 64 bytes, bare, + EOI and + RST0 + EOI.  stb reads a byte past the end of its buffer
    as 0, so an FF in the last byte is data to it, where the host decoder takes it for the start of a marker.  Either way
    only zero bits follow.  stb also needs a marker after the scan: a stream ending in FF has none, and after `FF FF D9` or
    `FF FF D0 FF D9` stb has taken both FFs and finds a stray D9 / D0.  So stb rejects every stream whose scan data ends in
    FF, and the two readings never make two different images.  Pinned here: wherever stb returns an image the host decoder
    returns the same bytes, and stb rejects every cut whose last scan byte is FF, with or without an RST / EOI after it.
    Cuts before the last restart interval are left out: decoding stops at the missing RSTn, and stb leaves the blocks it
    never decoded uninitialised."""
    n_ff = n_same = 0
    for i, (sampling, W, H, j, cases) in enumerate(truncation_cases()):
        last = j.resumes[-1] if j.resumes else j.scan_starts[0]
        cases = [(name, b) for name, b in cases if int(name[3:].split("+")[0]) >= last]
        p = write_container(tmp_path / f"t{i}.sens", [b for _, b in cases], W, H)
        _, host = host_colors(p, len(cases))
        ref = ref_colors(p, len(cases), W, H)
        for (name, b), h, r in zip(cases, host, ref):
            if j.data[int(name[3:].split("+")[0]) - 1] == 0xFF:
                n_ff += 1
                assert r is None, (sampling, name)
            if r is None: continue
            assert not isinstance(h, Exception) and (h == r).all(), (sampling, name)
            n_same += 1
    assert n_ff >= 30 and n_same > 200, (n_ff, n_same)


# ---- deflate stream families --------------------------------------------------------------------------------------------------
def pad_to(tokens, frame):
    """append literals so the stream holds at least `frame` bytes"""
    n = len(ds.decode_tokens(tokens))
    return tokens + [int(i * 7 & 255) for i in range(max(0, frame - n))]


def deflate_cases():
    """(name, zlib stream, the bytes it holds).  Every stream is checked against zlib.decompress as well."""
    rng = np.random.default_rng(5)
    out = []

    def add(name, d, tokens_or_data):
        raw = tokens_or_data if isinstance(tokens_or_data, bytes) else ds.decode_tokens(tokens_or_data)
        out.append((name, ds.zlib_stream(d.raw(), raw), raw))

    def lits(n, hi=256): return [int(x) for x in rng.integers(0, hi, n)]

    # dist = 32768 at the first output position where it is legal, lengths 3, 32, 33, 258
    first = lits(32768)
    for ln in (3, 32, 33, 258):
        for kind in ("fixed", "dynamic"):
            toks = first + [(ln, 32768)] + [1, 2, 3]
            d = ds.Deflate(); getattr(d, kind)(toks, last=True); add(f"dist32768-len{ln}-{kind}", d, toks)
    # length-258 matches at distances 1..40, 63, 64, 65 (copies overlapping themselves, powers of two and others)
    for dist in list(range(1, 41)) + [63, 64, 65]:
        toks = lits(dist) + [(258, dist), (258, dist), 9, (100, dist)]
        d = ds.Deflate(); d.dynamic(toks, last=True); add(f"len258-dist{dist}", d, toks)
    # stored blocks: across the 32 KB ring wrap, LEN 0, LEN 65535, and one after a dynamic block at an odd bit position
    a, b = bytes(lits(30000)), bytes(lits(6000))
    d = ds.Deflate(); d.stored(a); d.stored(b); d.stored(b"", last=True); add("stored-ring-wrap-len0", d, a + b)
    big = bytes(lits(65535))
    d = ds.Deflate(); d.stored(big); d.fixed([(258, 32768)], last=True); add("stored-65535-then-match", d, ds.decode_tokens(list(big) + [(258, 32768)]))
    for extra in range(16):
        toks = lits(999 + extra, 4) + [(5, 3)]
        d = ds.Deflate(); d.dynamic(toks)
        if d.bits.n % 2 == 1: break
    assert d.bits.n % 2 == 1
    tail = bytes(range(200)); d.stored(tail, last=True); add("dynamic-then-stored-odd-bit", d, ds.decode_tokens(toks) + tail)
    # HLIT 257 / HDIST 1 with a single distance code (an incomplete code), and HLIT 286 / HDIST 30
    toks = lits(600)
    d = ds.Deflate(); d.dynamic(toks, last=True, dist_lens=[1], hlit=257, hdist=1); add("hlit257-hdist1-one-code", d, toks)
    d = ds.Deflate(); d.dynamic(toks + [(9, 5)], last=True, dist_lens=[0, 0, 0, 0, 1], hdist=5); add("one-distance-code-of-five", d, toks + [(9, 5)])
    toks2 = toks + [(258, 1), (10, 7), (3, 513)]
    d = ds.Deflate(); d.dynamic(toks2, last=True, hlit=286, hdist=30); add("hlit286-hdist30", d, toks2)
    # 15-bit literal/length codes and distance codes longer than the lookahead (10 bits for literal/length, 8 for distance):
    # a chain of lengths 1, 2, ..., n-1, n-1 over 16 literal/length symbols and 11 distance symbols
    lsyms = [256, 257] + list(range(11)) + [258, 11, 12]            # 12 and 258 get the two 15-bit codes
    ll = [0] * 286
    for i, sy in enumerate(lsyms): ll[sy] = min(i + 1, 15)
    dsyms = list(range(9)) + [21, 29]                                 # 21 and 29 get the two 10-bit codes
    dl = [0] * 30
    for i, sy in enumerate(dsyms): dl[sy] = min(i + 1, 10)
    toks3 = lits(30000, 13) + [(3, 1), (4, 2000), (3, 24577)] * 40 + [12] * 50 + [(4, 24577), (4, 1600)] * 30
    d = ds.Deflate(); d.dynamic(toks3, last=True, lit_lens=ll, dist_lens=dl); add("15-bit-codes", d, toks3)
    # repeat code 16 running from the literal/length lengths into the distance lengths, and repeat code 18 with a run of 138:
    # 16 literal/length codes and 16 distance codes, all 4 bits
    ll = [0] * 286
    for sy in list(range(12)) + [256, 283, 284, 285]: ll[sy] = 4
    dl = [4] * 16
    cl = [(4, 0, 0)] * 12 + [(18, 7, 127), (18, 7, 95), (4, 0, 0), (18, 7, 15), (4, 0, 0), (16, 2, 1), (16, 2, 3), (16, 2, 3), (4, 0, 0), (4, 0, 0)]
    toks4 = lits(100, 12) + [(258, 1), (200, 2), (230, 3), (199, 17)] + lits(50, 12)
    d = ds.Deflate(); d.dynamic(toks4, last=True, lit_lens=ll, dist_lens=dl, hlit=286, hdist=16, cl_syms=cl); add("repeat16-crossing-repeat18-138", d, toks4)
    # 2,000 one-symbol blocks at the start of one 640x480 depth frame, the rest in stored blocks
    d = ds.Deflate(); body = bytearray()
    for i in range(2000):
        v = i & 255 if i % 2 else (i * 7) & 255
        (d.fixed if i % 2 else d.dynamic)([v]); body.append(v)
    rest = bytes((np.arange(640 * 480 * 2 - len(body)) * 13 & 255).astype(np.uint8))
    for k in range(0, len(rest), 65535): d.stored(rest[k:k + 65535], last=k + 65535 >= len(rest))
    add("2000-one-symbol-blocks", d, bytes(body) + rest)
    return out


def deflate_errors():
    """(name, zlib stream) that zlib and every inflate path here must reject"""
    rng = np.random.default_rng(6)
    toks = [int(x) for x in rng.integers(0, 256, 300)]
    ll, _ = ds.lengths_from_tokens(toks)
    out = []
    over = list(ll); over[0] = over[1] = over[2] = 1                    # three 1-bit codes: over-subscribed
    d = ds.Deflate(); d.dynamic([], last=True, lit_lens=over, dist_lens=[1]); out.append(("over-subscribed", d))
    sent = list(ll[:257]) + [1]
    d = ds.Deflate(); d.dynamic([], last=True, lit_lens=ll, dist_lens=[1], hlit=257, hdist=1, cl_syms=[(16, 2, 0)] + ds.rle_lengths(sent))
    out.append(("repeat16-first", d))
    d = ds.Deflate(); d.dynamic([], last=True, lit_lens=[8] * 256, dist_lens=[1]); out.append(("no-end-of-block", d))
    d = ds.Deflate(); d.stored(b"abc" * 10, last=True, nlen=0x1234); out.append(("nlen-not-len-complement", d))
    d = ds.Deflate(); d.fixed(toks[:100] + [(5, 101)], last=True); out.append(("distance-before-start", d))
    return [(name, ds.zlib_stream(d.raw(), b"")) for name, d in out]


@pytest.mark.parametrize("case", range(len(deflate_cases())), ids=[c[0] for c in deflate_cases()])
def test_crafted_deflate_matches_zlib_and_host_inflate(built, case):
    name, z, raw = deflate_cases()[case]
    assert zlib.decompress(z) == raw, name
    assert sens.inflate_host(z, len(raw)) == raw, name


@pytest.mark.parametrize("case", range(len(deflate_errors())), ids=[c[0] for c in deflate_errors()])
def test_malformed_deflate_is_an_error(built, case):
    name, z = deflate_errors()[case]
    with pytest.raises(zlib.error):
        zlib.decompress(z)
    with pytest.raises(ScnError):
        sens.inflate_host(z, 1000)
