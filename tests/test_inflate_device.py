"""The GPU inflate (csrc/inflate.cu) through its public paths: ChunkedVariable.load_device,
Cutout.to_device() of lazily loaded cutouts, and Deflate GeoTIFF segments.  Every expected value
comes from Python's zlib or from the host decoder (ChunkedVariable.load / isel_time), and is
compared bit for bit."""

import os
import struct
import zlib

import numpy as np
import pytest

import atlite_b200 as ab
from atlite_b200 import _lib, convert, engine, geotiff, ingest, synthetic as syn

gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------
# zlib streams: encoders and hand-built blocks
# ---------------------------------------------------------------------------------------------


class BitWriter:
    """Deflate's LSB-first bit packing."""

    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def bits(self, v, k):
        self.acc |= (v & ((1 << k) - 1)) << self.n
        self.n += k
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def code(self, code, length):  # Huffman codes go MSB-first
        self.bits(int(format(code, f"0{length}b")[::-1], 2), length)

    def align(self):
        if self.n:
            self.bits(0, 8 - self.n)

    def zlib(self, payload):
        self.align()
        return b"\x78\x01" + bytes(self.out) + struct.pack(">I", zlib.adler32(payload))


def canonical(lens):
    """Canonical Huffman codes {symbol: (code, length)} of a length list (RFC 1951 3.2.2)."""
    count = np.bincount([v for v in lens if v], minlength=16)
    code, nxt = 0, {}
    for b in range(1, 16):
        code = (code + (count[b - 1] if b > 1 else 0)) << 1
        nxt[b] = code
    out = {}
    for s, v in enumerate(lens):
        if v:
            out[s] = (nxt[v], v)
            nxt[v] += 1
    return out


LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195,
            227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073,
             4097, 6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def dynamic_block(w, lit_lens, dist_lens, tokens, final=True, clen=None):
    """One dynamic block: code lengths sent one by one with a 16-symbol code-length code of
    4-bit codes (or ``clen``, the 19 code-length code lengths, to corrupt it); tokens are bytes
    (literals) or (length, distance) pairs."""
    nlen, ndist = len(lit_lens), len(dist_lens)
    w.bits(int(final), 1)
    w.bits(2, 2)
    w.bits(nlen - 257, 5)
    w.bits(ndist - 1, 5)
    w.bits(19 - 4, 4)
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    clen = [4] * 16 + [0, 0, 0] if clen is None else clen
    for s in order:
        w.bits(clen[s], 3)
    cc = canonical(clen)
    for v in list(lit_lens) + list(dist_lens):
        w.code(*cc[v])
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for t in tokens:
        if isinstance(t, int):
            w.code(*lc[t])
            continue
        length, dist = t
        s = max(i for i, b in enumerate(LEN_BASE) if b <= length)
        w.code(*lc[257 + s])
        w.bits(length - LEN_BASE[s], LEN_EXTRA[s])
        d = max(i for i, b in enumerate(DIST_BASE) if b <= dist)
        w.code(*dc[d])
        w.bits(dist - DIST_BASE[d], DIST_EXTRA[d])
    w.code(*lc[256])


def fixed_code(w, sym):
    if sym < 144:
        w.code(0x30 + sym, 8)
    elif sym < 256:
        w.code(0x190 + sym - 144, 9)
    elif sym < 280:
        w.code(sym - 256, 7)
    else:
        w.code(0xC0 + sym - 280, 8)


def expand(tokens):
    out = bytearray()
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            length, dist = t
            for _ in range(length):
                out.append(out[-dist])
    return bytes(out)


LONG_CODES = [0] * 257  # symbols 97..111 with code lengths 1..15, end-of-block 15: a complete code
for _k in range(15):
    LONG_CODES[97 + _k] = _k + 1
LONG_CODES[256] = 15


def hand_built():
    """{name: (stream, payload)} of streams zlib's encoder does not write."""
    out = {}
    # a dynamic block with a single distance code (incomplete, one code of length 1)
    lit = [0] * 266
    lit[97] = lit[98] = lit[99] = 2
    lit[256] = lit[265] = 3  # 265: lengths 11-12
    toks = [97, 98, 99] + [(11, 3)] * 9 + [97]  # 3 + 99 + 1 = 103 ... padded below
    toks += [97] * (-len(expand(toks)) % 4)
    w = BitWriter()
    dynamic_block(w, lit, [0, 0, 1], toks)
    out["single distance code"] = (w.zlib(expand(toks)), expand(toks))
    # a literal-only block whose distance tree has no code at all
    lit = [0] * 257
    lit[97] = lit[98] = lit[99] = 2
    lit[100] = lit[256] = 3
    toks = list(np.random.default_rng(5).choice([97, 98, 99, 100], 400))
    toks = [int(t) for t in toks]
    w = BitWriter()
    dynamic_block(w, lit, [0], toks)
    out["empty distance tree"] = (w.zlib(expand(toks)), expand(toks))
    # length-258 matches (symbol 285) at distance 1
    lit = [0] * 286
    lit[120] = 1
    lit[256] = lit[285] = 2
    toks = [120] + [(258, 1)] * 31 + [120] * 1  # 1 + 7998 + 1 = 8000 bytes
    w = BitWriter()
    dynamic_block(w, lit, [1], toks)
    out["symbol 285"] = (w.zlib(expand(toks)), expand(toks))
    # a fixed block, then a dynamic one: the decoder rebuilds its tables between blocks
    w = BitWriter()
    w.bits(0, 1)
    w.bits(1, 2)
    for c in b"fixed!!!":
        fixed_code(w, c)
    fixed_code(w, 256)
    lit = [0] * 257
    lit[97] = lit[98] = lit[99] = 2
    lit[100] = lit[256] = 3
    dynamic_block(w, lit, [0], [97, 98, 99, 100])
    out["fixed then dynamic"] = (w.zlib(b"fixed!!!abcd"), b"fixed!!!abcd")
    # literal/length codes of 11-15 bits: decoded past the 10-bit root table
    toks = [int(t) for t in np.random.default_rng(6).choice(np.arange(97, 112), 4000)]
    toks += [111] * (-len(toks) % 4)
    w = BitWriter()
    dynamic_block(w, LONG_CODES, [0], toks)
    out["codes of 11-15 bits"] = (w.zlib(expand(toks)), expand(toks))
    for name, (stream, payload) in out.items():
        assert zlib.decompress(stream) == payload, name  # the construction is valid zlib
    return out


def encoders():
    """{name: encode(payload) -> zlib stream}: levels, strategies, window sizes and flushes."""
    def enc(level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY, flush=None, every=0):
        def f(data):
            c = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
            if flush is None:
                return c.compress(data) + c.flush()
            out = b""
            for i in range(0, len(data), every):
                out += c.compress(data[i:i + every]) + c.flush(flush)
            return out + c.flush()
        return f

    out = {f"level {lv}": enc(lv) for lv in (0, 1, 6, 9)}
    out.update({f"strategy {s}": enc(6, strategy=getattr(zlib, s))
                for s in ("Z_FIXED", "Z_HUFFMAN_ONLY", "Z_RLE", "Z_FILTERED")})
    out.update({f"wbits {wb}": enc(9, wbits=wb) for wb in range(9, 16)})
    out["sync flush"] = enc(6, flush=zlib.Z_SYNC_FLUSH, every=1000)
    out["full flush"] = enc(9, flush=zlib.Z_FULL_FLUSH, every=777)
    out["stored sync flush"] = enc(0, flush=zlib.Z_SYNC_FLUSH, every=3000)
    return out


def payloads(size=1 << 16):
    """{name: bytes} of one size: constant, random, periodic (periods 1-40), far matches, floats."""
    rng = np.random.default_rng(11)
    out = {"constant": b"\x07" * size, "random": rng.bytes(size)}
    for p in range(1, 41):
        out[f"period {p}"] = (rng.bytes(p) * (size // p + 1))[:size]
    half = rng.bytes(size // 2)
    out["far matches"] = half + half  # length-258 matches at distance 32768
    y, x = np.mgrid[0:64, 0:256]
    field = (280.0 + 5.0 * np.sin(x / 17.0) * np.cos(y / 11.0) + rng.normal(0, 0.01, (64, 256))).astype(np.float32)
    out["shuffled float32"] = ingest.shuffle_bytes(field)
    return out


def stream_variable(path, streams, nbytes):
    """A ChunkedVariable whose chunk t is zlib stream t, each decoding to ``nbytes`` (a multiple of 4)
    bytes read as '<f4' -- the raw bits come back unchanged."""
    offs, sizes = [], []
    with open(path, "wb") as fh:
        for s in streams:
            offs.append(fh.tell())
            sizes.append(len(s))
            fh.write(s)
    n = nbytes // 4
    return ingest.ChunkedVariable(path, (len(streams), 1, n), (1, 1, n), "<f4", offs, sizes,
                                  [[t, 0, 0] for t in range(len(streams))], shuffle=False, deflate=True)


def device_bytes(var):
    return var.load_device(0, var.shape[0]).view(__import__("torch").int32).cpu().numpy().view(np.uint8)


# ---------------------------------------------------------------------------------------------
# 1. decoder against zlib
# ---------------------------------------------------------------------------------------------


def test_hand_built_streams_are_zlib():
    """CPU: the test's own block writer makes streams zlib decodes to the intended payloads."""
    assert len(hand_built()) == 5
    assert max(LONG_CODES) > 10 and sum(2.0 ** -v for v in LONG_CODES if v) == 1.0  # the slow path is taken


def test_load_device_checks_the_window(tmp_path):
    """CPU: a window past the variable's steps, rows or columns is refused before any device work."""
    var = stream_variable(tmp_path / "w.bin", [zlib.compress(bytes(64))] * 2, 64)
    for lo, hi, rows, cols in ((0, 3, None, None), (-1, 1, None, None), (0, 1, (0, 2), None), (0, 1, None, (3, 20))):
        with pytest.raises(ValueError, match="outside the variable"):
            var.load_device(lo, hi, rows, cols, device=0)


@gpu
def test_encoders_and_payloads_bitwise(tmp_path):
    pays, encs = payloads(), encoders()
    streams, want = [], []
    for pn, p in pays.items():
        for en, e in encs.items():
            s = e(p)
            assert zlib.decompress(s) == p, (pn, en)
            streams.append(s)
            want.append(p)
    var = stream_variable(tmp_path / "s.bin", streams, len(want[0]))
    got = device_bytes(var).reshape(len(streams), -1)
    bad = [i for i in range(len(streams)) if got[i].tobytes() != want[i]]
    assert not bad, [(list(pays)[i // len(encs)], list(encs)[i % len(encs)]) for i in bad[:10]]
    # one chunk per batch: the same bits
    var.device_batch_bytes = 1
    assert np.array_equal(device_bytes(var).reshape(len(streams), -1), got)


@gpu
@pytest.mark.parametrize("name", ["single distance code", "empty distance tree", "symbol 285", "fixed then dynamic",
                                  "codes of 11-15 bits"])
def test_hand_built_streams(tmp_path, name):
    stream, payload = hand_built()[name]
    assert len(payload) % 4 == 0  # the chunk holds whole float32 elements
    var = stream_variable(tmp_path / "h.bin", [stream, stream], len(payload))
    got = device_bytes(var).reshape(2, -1)
    assert got[0].tobytes() == payload and got[1].tobytes() == payload


# ---------------------------------------------------------------------------------------------
# 2. corrupt input is reported, not faulted
# ---------------------------------------------------------------------------------------------


def _fixed(tokens_fn):
    w = BitWriter()
    w.bits(1, 1)
    w.bits(1, 2)
    tokens_fn(w)
    return w


def corrupt_cases():
    good_payload = bytes(range(64))
    good = zlib.compress(good_payload, 9)
    cases = {}
    cases["bad zlib header"] = b"\x78\x02" + good[2:]
    cases["preset dictionary"] = b"\x78\x20" + b"\x00\x00\x00\x01" + good[2:]
    w = BitWriter()
    w.bits(1, 1)
    w.bits(3, 2)
    cases["invalid block type"] = w.zlib(good_payload)
    cases["stored block length"] = b"\x78\x01\x01" + struct.pack("<HH", 64, 0x1234) + good_payload
    w = BitWriter()
    lit = [0] * 257
    lit[97] = lit[256] = 1
    dynamic_block(w, lit, [0], [97], clen=[1] * 19)  # 19 one-bit codes: over-subscribed
    cases["invalid code-length set"] = w.zlib(b"a")

    def sym286(w):
        fixed_code(w, 97)
        fixed_code(w, 286)
    cases["symbol (286)"] = _fixed(sym286).zlib(good_payload)

    def dist30(w):
        fixed_code(w, 97)
        fixed_code(w, 97)
        fixed_code(w, 257)
        w.code(30, 5)
    cases["symbol (dist 30)"] = _fixed(dist30).zlib(good_payload)

    def too_far(w):
        fixed_code(w, 97)
        fixed_code(w, 257)
        w.code(1, 5)  # distance 2 after one byte
        fixed_code(w, 256)
    cases["distance too far back"] = _fixed(too_far).zlib(good_payload)
    cases["truncated"] = good[:len(good) // 2]
    cases["Adler-32"] = good[:-1] + bytes([good[-1] ^ 1])
    cases["output longer"] = zlib.compress(good_payload + b"more", 9)
    cases["output shorter"] = zlib.compress(good_payload[:-4], 9)
    cases["output shorter (empty)"] = zlib.compress(b"", 9)
    return good, good_payload, cases


REASONS = {"bad zlib header": "bad zlib header", "preset dictionary": "preset dictionary",
           "invalid block type": "invalid block type", "stored block length": "stored block length",
           "invalid code-length set": "invalid code-length set", "symbol (286)": "invalid literal/length or distance symbol",
           "symbol (dist 30)": "invalid literal/length or distance symbol",
           "distance too far back": "distance too far back", "truncated": "truncated", "Adler-32": "Adler-32 mismatch",
           "output longer": "output longer", "output shorter": "output shorter",
           "output shorter (empty)": "output shorter"}


def test_corrupt_cases_are_rejected_by_zlib(tmp_path):
    """CPU: every corruption is one zlib rejects too, and the host decoder reports it as zlib."""
    good, payload, cases = corrupt_cases()
    assert set(cases) == set(REASONS)
    for name, s in cases.items():
        try:
            ok = zlib.decompress(s) == payload
        except zlib.error:
            ok = False
        assert not ok, name
        var = stream_variable(tmp_path / "c.bin", [good, s], len(payload))
        with pytest.raises(_lib.AtlError, match="zlib:"):
            var.load(0, 2)


@gpu
@pytest.mark.parametrize("name", sorted(REASONS))
def test_corrupt_chunk_raises(tmp_path, name):
    good, payload, cases = corrupt_cases()
    var = stream_variable(tmp_path / "c.bin", [good, cases[name], good], len(payload))
    with pytest.raises(_lib.AtlError, match=r"zlib: chunk at \(t, y, x\) = \(1, 0, 0\): .*" + REASONS[name]):
        var.load_device(0, 3)
    # the good chunks still decode, and the device is usable afterwards
    ok = stream_variable(tmp_path / "g.bin", [good, good], len(payload))
    assert device_bytes(ok).tobytes() == payload * 2


@gpu
@pytest.mark.parametrize("name", sorted(REASONS))
def test_corrupt_geotiff_segment_raises(tmp_path, name):
    """The same corruptions as GeoTIFF Deflate segments: ValueError naming the segment and the reason."""
    write_tiff, _ = _write_tiff()
    good, payload, cases = corrupt_cases()
    arr = np.frombuffer(payload * 3, np.uint8).reshape(3, 64)
    p = write_tiff(tmp_path / "c.tif", arr, tiled=False, block=(1, 0), compression=8, override={1: cases[name]})
    with pytest.raises(ValueError, match=r"segment 1: Deflate data is corrupt: .*" + REASONS[name]):
        geotiff.read(p)
    got = engine.GeoTiffOp()(geotiff.info(p), (0, 1), (0, 64)).cpu().numpy()  # the other segments decode
    assert got.tobytes() == payload


# ---------------------------------------------------------------------------------------------
# 3. the to_device contract
# ---------------------------------------------------------------------------------------------


def _bits(t):
    import torch

    return t.contiguous().view(torch.int32).cpu().numpy()


def _assert_contract(lazy, pad=True, variables=None):
    nt = len(lazy.coords["time"])
    want = ab.Cutout(data=lazy.isel_time(0, nt)).to_device(variables=variables, pad=pad)
    got = ab.Cutout(data=lazy).to_device(variables=variables, pad=pad)
    names = list(want.data.keys())
    assert names == list(got.data.keys())
    for n in names:
        a, b = want.data.raw(n), got.data.raw(n)
        assert a.shape == b.shape and a.dtype == b.dtype, (n, a.shape, b.shape)
        assert np.array_equal(_bits(a), _bits(b)), n


def _fields(nt, ny, nx, seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:ny, 0:nx]
    base = 280.0 + 8.0 * np.sin(x / 5.0)[None] * np.cos(y / 3.0)[None] + np.arange(nt)[:, None, None] * 0.01
    a = (base + rng.normal(0, 0.2, (nt, ny, nx))).astype(np.float32)
    a[:, 0, 0] = -0.0
    a[1, 1, 1] = np.nan
    a[2, 2, 2] = np.float32(1e-40)  # subnormal
    return a


def _packed_variable(tmp_path, name, arr, dtype, chunk, complevel, shuffle, scale=None, offset=None, fill=None,
                     drop=()):
    """A ChunkedVariable of ``arr`` stored as ``dtype`` with the container's encoding; chunk indices
    in ``drop`` are left out of the index (HDF5 leaves unwritten chunks out)."""
    p = ingest.write_chunked(tmp_path / f"{name}.bin", {name: arr.astype(dtype)}, {}, chunk=chunk,
                             complevel=complevel, shuffle=shuffle)
    import json

    with open(str(p) + ".index.json") as fh:
        v = json.load(fh)["variables"][name]
    keep = [i for i in range(len(v["offsets"])) if i not in set(drop)]
    return ingest.ChunkedVariable(p, v["shape"], v["chunk"], v["dtype"], np.asarray(v["offsets"])[keep],
                                  np.asarray(v["sizes"])[keep], np.asarray(v["origins"])[keep], v["shuffle"],
                                  v["deflate"], scale_factor=scale, add_offset=offset, fill_value=fill)


def _lazy_of(variables, nt, ny, nx):
    x, y = syn.make_coords(nx, ny, 5.0, 45.0, 0.25, 0.25)
    coords = dict(time=syn.make_time(nt), x=x, y=y, lon=x, lat=y)
    static = {"height": np.arange(ny * nx, dtype=np.float32).reshape(ny, nx)}
    return ingest._lazy(variables, coords, static, {}, 100)


NT, NY, NX = 23, 13, 17  # odd width: pad=True widens the rows to 20

CHUNKS = [(100, None, None), (7, 5, 6)]


@gpu
@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("shuffle", [True, False])
def test_to_device_dtypes_and_packing(tmp_path, chunk, shuffle):
    a = _fields(NT, NY, NX)
    i16 = np.round((a - 280.0) / 0.01).astype(np.float64)
    i16[np.isnan(i16)] = -32767
    i16[3, 4, 5] = -32767  # the fill value -> NaN
    i16[:, 0, 0] = 0
    nanpay = a.copy()
    nanpay.view(np.uint32)[4, 3, 2] = 0x7fa00001  # a signalling NaN payload through a converted float32
    variables = {
        "f4": _packed_variable(tmp_path, "f4", a, "<f4", chunk, 9, shuffle),
        "f4be": _packed_variable(tmp_path, "f4be", a, ">f4", chunk, 1, shuffle),
        "f8": _packed_variable(tmp_path, "f8", a.astype(np.float64) * 1.0000001, "<f8", chunk, 6, shuffle),
        "f8be": _packed_variable(tmp_path, "f8be", a.astype(np.float64), ">f8", chunk, 3, shuffle),
        "i2": _packed_variable(tmp_path, "i2", i16, "<i2", chunk, 9, shuffle, scale=0.01, offset=280.0, fill=-32767),
        "i2be": _packed_variable(tmp_path, "i2be", i16, ">i2", chunk, 5, shuffle, scale=np.float64(0.01),
                                 offset=np.float32(280.0), fill=np.int16(-32767)),
        "u2": _packed_variable(tmp_path, "u2", i16 + 40000, "<u2", chunk, 2, shuffle, scale=0.5, fill=40000.0),
        "i4": _packed_variable(tmp_path, "i4", i16 * 1000.0 + 123456789, "<i4", chunk, 4, shuffle, scale=1e-3),
        "f4fill": _packed_variable(tmp_path, "f4fill", nanpay, "<f4", chunk, 7, shuffle, fill=float(a[0, 1, 1]),
                                   scale=2.0, offset=-1.5),
        "f8fill": _packed_variable(tmp_path, "f8fill", a.astype(np.float64), "<f8", chunk, 8, shuffle,
                                   fill=float(a[5, 5, 5])),
    }
    lazy = _lazy_of(variables, NT, NY, NX)
    for pad in (True, False):
        _assert_contract(lazy, pad)


@gpu
@pytest.mark.parametrize("complevel", range(10))
def test_to_device_complevels(tmp_path, complevel):
    a = _fields(NT, NY, NX, seed=complevel)
    v = {"f": _packed_variable(tmp_path, "f", a, "<f4", (7, 5, 6), complevel, complevel % 2 == 0)}
    _assert_contract(_lazy_of(v, NT, NY, NX))


@gpu
@pytest.mark.parametrize("chunk", CHUNKS)
def test_to_device_missing_chunks_and_selections(tmp_path, chunk):
    a = _fields(NT, NY, NX, seed=3)
    i16 = np.round((a - 280.0) / 0.01)
    i16[np.isnan(i16)] = 0
    variables = {
        "f4": _packed_variable(tmp_path, "f4", a, "<f4", chunk, 9, True, drop=(1, 4)),
        "i2": _packed_variable(tmp_path, "i2", i16, "<i2", chunk, 9, True, scale=0.01, offset=280.0, fill=0,
                               drop=(0,)),
    }
    lazy = _lazy_of(variables, NT, NY, NX)
    _assert_contract(lazy)
    x, y, t = lazy.coords["x"], lazy.coords["y"], lazy.coords["time"]
    for sel in (dict(time=slice(t[3], t[17])), dict(x=slice(x[2], x[12]), y=slice(y[1], y[9])),
                dict(time=slice(t[8], t[8]), x=slice(x[5], x[5])),
                dict(time=slice(t[6], t[20]), x=slice(x[3], x[16]), y=slice(y[4], y[12]))):
        sub = ab.Cutout(data=lazy).sel(**sel).data
        _assert_contract(sub)
        if len(sub.coords["x"]) > 2:  # a selection of a selection
            _assert_contract(sub.sel(x=slice(sub.coords["x"][1], sub.coords["x"][-1])), pad=False)


@gpu
def test_to_device_one_chunk_per_batch(tmp_path):
    a = _fields(NT, NY, NX, seed=4)
    v = {"f": _packed_variable(tmp_path, "f", a, "<f4", (7, 5, 6), 9, True)}
    lazy = _lazy_of(v, NT, NY, NX)
    want = ab.Cutout(data=lazy).to_device().data.raw("f")
    v["f"].device_batch_bytes = 1
    got = ab.Cutout(data=lazy).to_device().data.raw("f")
    assert np.array_equal(_bits(want), _bits(got))
    _assert_contract(lazy)


@gpu
def test_to_device_netcdf3_host_parts(tmp_path, monkeypatch):
    from scipy.io import netcdf_file

    a = _fields(NT, NY, NX, seed=5).astype(np.float64)
    x, y = syn.make_coords(NX, NY, 5.0, 45.0, 0.25, 0.25)
    p = str(tmp_path / "c.nc")
    f = netcdf_file(p, "w")
    f.createDimension("time", NT)
    f.createDimension("y", NY)
    f.createDimension("x", NX)
    tv = f.createVariable("time", "f8", ("time",))
    tv[:] = np.arange(NT)
    tv.units = "hours since 2013-01-01"
    f.createVariable("x", "f8", ("x",))[:] = x
    f.createVariable("y", "f8", ("y",))[:] = y
    v = f.createVariable("temperature", "i2", ("time", "y", "x"))
    v[:] = np.round(np.nan_to_num(a - 280.0) * 100).astype(np.int16)
    v.scale_factor, v.add_offset = 0.01, 280.0
    f.createVariable("wnd100m", "f4", ("time", "y", "x"))[:] = a.astype(np.float32)
    f.close()
    lazy = ingest.open_cutout(p)
    monkeypatch.setattr(convert, "PART_BYTES", NY * NX * 4 * 5)  # parts of 5 steps
    _assert_contract(lazy)
    _assert_contract(lazy, pad=False)


# ---------------------------------------------------------------------------------------------
# 4. conversions agree
# ---------------------------------------------------------------------------------------------


@gpu
def test_conversions_on_a_device_decoded_raw_era5_cutout(tmp_path):
    nx, ny, nt = 37, 14, 60
    rng = np.random.default_rng(3)
    shp = (nt, ny, nx)
    f = lambda lo, hi: rng.uniform(lo, hi, shp).astype(np.float32)  # noqa: E731
    d = dict(u100=f(-15, 15), v100=f(-15, 15), u10=f(-8, 8), v10=f(-8, 8), fsr=f(-0.05, 2.0),
             ssrd=f(0, 3.0e6), tisr=f(0, 4.5e6), t2m=f(250, 305), stl4=f(270, 290), d2m=f(250, 295))
    d["ssr"] = (d["ssrd"] * rng.uniform(0.6, 1.0, shp)).astype(np.float32)
    d["fdir"] = (d["ssrd"] * rng.uniform(0.0, 1.1, shp)).astype(np.float32)
    x, y = syn.make_coords(nx, ny, -10.0, 35.0, 0.5, 0.5)
    t = syn.make_time(nt + 24 * 40)[24 * 40:]
    p = ingest.write_chunked(tmp_path / "raw.bin", d, dict(time=t, x=x, y=y), chunk=(16, 5, 9))
    lazy = ingest.open_cutout(p)
    host = ab.Cutout(data=lazy.isel_time(0, nt)).to_device()
    dev = ab.Cutout(data=lazy).to_device()
    m = syn.make_shapes(nx, ny, 7)
    prev = ab.set_deterministic(True)
    try:
        for method, kw in (("pv", dict(panel="CSi", orientation="latitude_optimal")),
                           ("wind", dict(turbine="Vestas_V112_3MW")), ("heat_demand", dict())):
            a = getattr(host, method)(matrix=m, aggregate_time=None, **kw)
            b = getattr(dev, method)(matrix=m, aggregate_time=None, **kw)
            assert np.array_equal(np.asarray(a.values), np.asarray(b.values), equal_nan=True), method
    finally:
        ab.set_deterministic(prev)


# ---------------------------------------------------------------------------------------------
# 5. Deflate GeoTIFFs
# ---------------------------------------------------------------------------------------------


def _write_tiff():
    import importlib.util

    spec = importlib.util.spec_from_file_location("_tiff_writer", os.path.join(os.path.dirname(__file__),
                                                                                "test_geotiff.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.write_tiff, mod._content


@gpu
@pytest.mark.parametrize("predictor", [1, 2, 3])
@pytest.mark.parametrize("tiled", [True, False])
def test_deflate_geotiff_segments(tmp_path, predictor, tiled):
    write_tiff, content = _write_tiff()
    rng = np.random.default_rng(predictor)
    dt = np.dtype("f4") if predictor == 3 else np.dtype("u2")
    arr = content(rng, (300, 290), dt, "blocky") if dt.kind == "u" else \
        (rng.normal(0, 1, (300, 290)).cumsum(1) * 10).astype(np.float32)
    block = (32, 48) if tiled else (3, 0)
    for bo in ("<", ">"):
        p = write_tiff(tmp_path / f"d{bo == '>'}.tif", arr, tiled=tiled, block=block, compression=8,
                       predictor=predictor, bo=bo)
        inf = geotiff.info(p)
        op = engine.GeoTiffOp(batch_bytes=20000)
        got = op(inf, (0, 300), (0, 290)).cpu().numpy()
        assert np.array_equal(got.view(np.uint8), arr.astype(arr.dtype.newbyteorder("=")).view(np.uint8)), bo
        assert op.stats["segments"] > 20 and op.stats["xfer_bytes"] == op.stats["stored_bytes"]
        win = op(inf, (17, 250), (5, 201)).cpu().numpy()
        assert np.array_equal(win.view(np.uint8), np.ascontiguousarray(arr[17:250, 5:201]).view(np.uint8))
