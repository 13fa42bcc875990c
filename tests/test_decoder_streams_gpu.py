"""GPU: the hand-built JPEG and deflate streams of test_decoder_streams_cpu.py through the warp-per-frame device decoders.

JPEG (jpeg_gpu.cu): the device output must be the host decoder's bytes (and stb's, where the reference library is built),
and for every stream of the class the device handles, the device must have decoded every frame itself (k == n), so a silent
fall-back to the host cannot hide a regression.  Deflate (inflate.cu): zlib's bytes with the window in shared memory and in
HBM, and the same errors as the host build."""
import zlib

import numpy as np
import pytest
import torch

import deflate_streams as ds
import jpeg_streams as js
import test_decoder_streams_cpu as cpu
from scannet_b200 import ScnError, sens

pytestmark = pytest.mark.gpu


def device_decode(jpegs, W, H, lut=None):
    """(device RGB8 frames, frames the device decoded itself)"""
    n = len(jpegs)
    if lut is None:
        out = torch.zeros((n, H, W, 3), dtype=torch.uint8, device="cuda")
        k = sens.jpeg_decode_batch_device(jpegs, W, H, out.data_ptr())
    else:
        d_lut = torch.from_numpy(lut).cuda()
        out = torch.zeros((n, len(lut), 3), dtype=torch.uint8, device="cuda")
        k = sens.jpeg_decode_batch_device(jpegs, W, H, out.data_ptr(), d_lut.data_ptr(), len(lut))
    return out.cpu().numpy(), k


def check(tmp_path, name, jpegs, W, H, all_on_device=True, stb=True):
    """device == host (== stb where built); the .sens entry point gives the same; k == n for the supported class"""
    p = cpu.write_container(tmp_path / f"{name}.sens", jpegs, W, H)
    s, host = cpu.host_colors(p, len(jpegs))
    for i, h in enumerate(host):
        assert not isinstance(h, Exception), (name, i, h)
    host = np.stack(host)
    ref = cpu.ref_colors(p, len(jpegs), W, H) if stb else None
    if ref is not None:
        for i, r in enumerate(ref):
            assert r is not None and (r == host[i]).all(), (name, i)
    got, k = device_decode(jpegs, W, H)
    for i in range(len(jpegs)):
        assert (got[i] == host[i]).all(), f"{name}[{i}]: device differs from the host decoder"
    if all_on_device: assert k == len(jpegs), f"{name}: the device declined {len(jpegs) - k} of {len(jpegs)} frames"
    out2 = torch.zeros((len(jpegs), H, W, 3), dtype=torch.uint8, device="cuda")
    assert s.decode_color_device(0, len(jpegs), out2.data_ptr()) == k
    assert (out2.cpu().numpy() == host).all()
    return host, k


def same_bytes_or_same_error(tmp_path, name, jpegs, W, H):
    """damaged streams, one call each: the device path gives the host decoder's bytes, or fails where it fails"""
    p = cpu.write_container(tmp_path / f"{name}.sens", jpegs, W, H)
    _, host = cpu.host_colors(p, len(jpegs))
    for i, (b, h) in enumerate(zip(jpegs, host)):
        if isinstance(h, Exception):
            with pytest.raises(ScnError):
                device_decode([b], W, H)
        else:
            got, _ = device_decode([b], W, H)
            assert (got[0] == h).all(), (name, i)


@pytest.mark.parametrize("sampling", list(cpu.SAMPLINGS))
def test_layouts_and_tables(tmp_path, built, sampling):
    jpegs = [s for kind in ("std", "optimal", "long16", "fast9_10") for _, s in cpu.layout_streams(sampling, kind)]
    check(tmp_path, sampling, jpegs, 41, 27)


@pytest.mark.parametrize("sampling", list(cpu.SAMPLINGS))
def test_coefficient_edges(tmp_path, built, sampling):
    check(tmp_path, sampling, [s for _, s in cpu.coefficient_streams(sampling)], 48, 32)


@pytest.mark.parametrize("sampling", ["420", "444", "grey"])
def test_stuffing_at_every_offset(tmp_path, built, sampling):
    """FF 00 at raw offsets 0..31 from the scan start and from every RSTn resume point"""
    streams = cpu.stuffing_streams(sampling)
    for name, j, t in streams:
        assert all(j.data[r + t] == 0xFF and j.data[r + t + 1] == 0 for r in j.scan_starts + j.resumes), name
    check(tmp_path, sampling, [j.data for _, j, _ in streams], 64, 48)


@pytest.mark.parametrize("sampling,W,H", [("420", 200, 40), ("422", 72, 24), ("444", 40, 24), ("440", 24, 40), ("grey", 96, 16)])
def test_restart_intervals(tmp_path, built, sampling, W, H):
    check(tmp_path, sampling, [s for _, s in cpu.restart_streams(sampling, W, H)], W, H)


def test_restart_markers_with_fill_bytes(tmp_path, built):
    """FF fill before every RSTn (T.81 B.1.1.2 allows it before any marker): the host decoder skips it and the device may
    hand such a frame to the host, with the same bytes.  stb v2.08 takes the first fill byte for the marker and stops
    decoding at the interval, so it is not compared here."""
    jpegs = [cpu.simple_stream(40, 24, s, seed=3, restart=2, rst_fill=2).data for s in ("420", "grey")]
    check(tmp_path, "rstfill", jpegs, 40, 24, all_on_device=False, stb=False)


@pytest.mark.parametrize("wh", [(496, 16), (497, 17), (511, 9), (512, 16), (528, 23), (1, 1), (1, 37), (37, 1), (33, 19)])
@pytest.mark.parametrize("sampling", ["420", "422", "440", "444", "grey"])
def test_sizes(tmp_path, built, wh, sampling):
    W, H = wh
    check(tmp_path, f"{sampling}-{W}x{H}", [cpu.simple_stream(W, H, sampling, seed=W + H + i).data for i in range(2)], W, H)


def test_grey_with_a_2x2_sampling_factor(tmp_path, built):
    """A one-component frame is coded as a non-interleaved scan whatever its sampling factors say: one block per MCU, rows
    of ceil(W / 8) blocks (T.81 A.2.2), which is how the host decoder and stb read it."""
    W, H = 40, 24
    jpegs = [cpu.simple_stream(W, H, comps=[js.Comp(1, h, v, 0, 0, 0)], seed=i).data for i, (h, v) in enumerate([(2, 2), (2, 1), (1, 2)])]
    check(tmp_path, "grey22", jpegs, W, H)


def test_scannet_colour_size_single_segments(tmp_path, built):
    """1296x968 with one DQT and one DHT segment, full frame and through a depth-registered map"""
    W, H = 1296, 968
    jpegs = [cpu.simple_stream(W, H, "420", seed=i, one_dqt=True, one_dht=True).data for i in range(2)]
    host, _ = check(tmp_path, "scannet", jpegs, W, H)
    rng = np.random.default_rng(2)
    lut = rng.integers(-1, W * H, 640 * 480).astype(np.int32); lut[:5] = [-1, 0, W * H - 1, W - 1, W * (H - 1)]
    got, k = device_decode(jpegs, W, H, lut)
    assert k == 2
    want = host.reshape(2, W * H, 3)[:, np.maximum(lut, 0)]; want[:, lut < 0] = 0
    assert (got == want).all()


def test_many_table_sets_in_one_batch(tmp_path, built):
    """240 frames, each with its own quantisation and optimal Huffman tables, mixed samplings of one size"""
    W, H = 48, 32
    rng = np.random.default_rng(9)
    jpegs = []
    for i in range(240):
        sampling = ["420", "422", "444", "440", "grey"][i % 5]
        comps = cpu.comps_for(sampling)
        blocks = js.random_blocks(rng, js.block_grid(W, H, comps), ac_max=int(rng.integers(5, 80)))
        restart = int(rng.integers(0, 4))
        dc, ac = cpu.table_kind("optimal", comps, blocks, restart=restart)
        quant = {c.tq: rng.integers(1, 60, 64) for c in comps}
        jpegs.append(js.write_jpeg(W, H, comps, blocks, quant, dc, ac, restart=restart).data)
    check(tmp_path, "batch", jpegs, W, H)


def test_declined_streams(tmp_path, built):
    """progressive, 4:1:1, Huffman table id 2, SOS order unlike SOF, three non-interleaved scans: the host decodes them (same
    bytes, and stb's), the device count leaves them out; 16-bit DQT is an error on both paths"""
    cv2 = pytest.importorskip("cv2")
    W, H = 48, 32
    img = np.random.default_rng(1).integers(0, 256, (H, W, 3)).astype(np.uint8)
    prog = cv2.imencode(".jpg", img, [int(cv2.IMWRITE_JPEG_PROGRESSIVE), 1])[1].tobytes()
    declined = [prog] + [s for _, s in cpu.declined_streams(W, H)]
    good = [cpu.simple_stream(W, H, "420", seed=i).data for i in range(2)]
    jpegs = [good[0]] + declined + [good[1]]
    p = cpu.write_container(tmp_path / "d.sens", jpegs, W, H)
    _, host = cpu.host_colors(p, len(jpegs))
    got, k = device_decode(jpegs, W, H)
    assert k == 2
    assert all((got[i] == host[i]).all() for i in range(len(jpegs)))
    with pytest.raises(ScnError):
        device_decode([good[0], cpu.dqt16_stream(W, H)], W, H)


def test_damaged_streams(tmp_path, built):
    """a code missing from the Huffman table, a DHT marker in the middle of the scan, and cuts at each of the last 64 bytes
    of scans with and without restart intervals: same bytes or same error as the host decoder"""
    W, H = 64, 48
    comps = cpu.comps_for("420")
    blocks = js.random_blocks(np.random.default_rng(4), js.block_grid(W, H, comps))
    t = js.std_tables()
    q = js.std_quant(1)
    # the DHT written for AC table 0 lacks the code of symbol 0x01 (so every coded 0x01 is an invalid code)
    ac0 = js.Huff(t["ac"][0].bits, t["ac"][0].vals)
    hole = js.crafted({s: ln for s, (_, ln) in ac0.code.items() if s != 0x01})
    missing = js.write_jpeg(W, H, comps, blocks, {0: q[0], 1: q[1]}, {0: t["dc"][0], 1: t["dc"][1]}, {0: t["ac"][0], 1: t["ac"][1]},
                            header_ac={0: hole, 1: t["ac"][1]}).data
    j = cpu.simple_stream(W, H, "420", seed=11)
    mid = (j.scan_starts[0] + len(j.data)) // 2
    dht = js.segment(0xC4, bytes([0x10]) + t["ac"][0].spec())
    mid_dht = j.data[:mid] + dht + j.data[mid:]
    cases = [missing, mid_dht]
    for _, _, _, jj, cuts in cpu.truncation_cases():
        cases += [b for _, b in cuts]
    same_bytes_or_same_error(tmp_path, "damaged", cases, W, H)


# ---- deflate -------------------------------------------------------------------------------------------------------------------
def inflate_device(streams, frame):
    out = torch.zeros((len(streams), frame), dtype=torch.uint8, device="cuda")
    sens.inflate_batch_device(streams, frame, out.data_ptr())
    return out.cpu().numpy()


@pytest.mark.parametrize("window", ["ring", "hbm"])
def test_crafted_deflate_on_device(built, window, monkeypatch):
    """every crafted stream, its frame exactly the bytes it holds, and with a final match / stored block that crosses the
    end of the frame (the output is cut at the frame size)"""
    monkeypatch.setenv("SCN_INFLATE_WINDOW", window)
    for name, z, raw in cpu.deflate_cases():
        assert inflate_device([z], len(raw))[0].tobytes() == raw, name
    rng = np.random.default_rng(3)
    lits = [int(x) for x in rng.integers(0, 256, 5000)]
    for tail in ([(258, 1)], [(258, 300)], [(40, 7)]):
        toks = lits + tail
        raw = ds.decode_tokens(toks)
        for kind in ("fixed", "dynamic"):
            d = ds.Deflate(); getattr(d, kind)(toks, last=True)
            z = ds.zlib_stream(d.raw(), raw)
            for cut in (1, tail[0][0] // 2, tail[0][0] - 1):
                assert inflate_device([z], len(raw) - cut)[0].tobytes() == raw[:-cut], (tail, kind, cut)
    d = ds.Deflate(); body = bytes(lits); d.fixed(lits[:100]); d.stored(body, last=True)
    raw = bytes(lits[:100]) + body
    assert inflate_device([ds.zlib_stream(d.raw(), raw)], len(raw) - 777)[0].tobytes() == raw[:-777]
    assert sens.inflate_last_timings()[2] == (window == "ring")


@pytest.mark.parametrize("window", ["ring", "hbm"])
def test_crafted_deflate_errors_on_device(built, window, monkeypatch):
    """over-subscribed code, repeat 16 first, no end-of-block code, NLEN != ~LEN, a distance before the start: errors on the
    host build and on the device; dist = o + 1 at the first legal position of dist = 32768 likewise"""
    monkeypatch.setenv("SCN_INFLATE_WINDOW", window)
    frame = 40000                                                   # larger than any of these streams holds: the error comes first
    good = zlib.compress(bytes(frame))
    lits = [int(x) for x in np.random.default_rng(2).integers(0, 256, 32768)]
    d = ds.Deflate(); d.fixed(lits[:32767] + [(3, 32768)], last=True)
    errors = cpu.deflate_errors() + [("dist-o+1", ds.zlib_stream(d.raw(), b""))]
    for name, z in errors:
        with pytest.raises(ScnError):
            sens.inflate_host(z, frame)
        with pytest.raises(ScnError, match="frame 1: corrupt"):
            inflate_device([good, z + bytes(2000), good], frame)


def test_batch_of_600_streams(built):
    """640 streams in one launch, crafted (fixed, dynamic, stored, mixed) and zlib, compressed lengths of every residue mod 4
    and mod 16 (the device reader loads aligned 32-bit words; streams are packed at 16-byte offsets)"""
    frame = 4096
    rng = np.random.default_rng(8)
    streams, want = [], []
    for i in range(640):
        raw_toks = []
        while len(ds.decode_tokens(raw_toks)) < frame:
            if raw_toks and rng.random() < 0.3:
                n = len(ds.decode_tokens(raw_toks))
                raw_toks.append((int(rng.integers(3, 259)), int(rng.integers(1, min(n, 32768) + 1))))
            else:
                raw_toks.append(int(rng.integers(0, 256 if i % 3 else 8)))
        raw = ds.decode_tokens(raw_toks)
        kind = i % 5
        if kind == 4:
            z = zlib.compress(raw, int(rng.integers(0, 10)))
        else:
            d = ds.Deflate()
            if kind == 0: d.fixed(raw_toks, last=True)
            elif kind == 1: d.dynamic(raw_toks, last=True)
            elif kind == 2: d.stored(raw[:1000]); d.stored(raw[1000:], last=True)
            else:
                h = len(raw_toks) // 2
                d.dynamic(raw_toks[:h]); d.stored(b"", last=False); d.fixed(raw_toks[h:], last=True)
            z = ds.zlib_stream(d.raw(), raw)
            z = z + bytes(int(rng.integers(0, 4)))                    # trailing bytes after the stream: lengths of every residue
        streams.append(z); want.append(raw[:frame])
    assert {len(z) % 4 for z in streams} == {0, 1, 2, 3} and len({len(z) % 16 for z in streams}) == 16
    got = inflate_device(streams, frame)
    for i in range(len(streams)):
        assert got[i].tobytes() == want[i], i
