"""GeoTIFF reader (atlite_b200/geotiff.py, csrc/geotiff.cu): the IFD parser, windows and refusals on
the CPU; the GPU decode bitwise against libtiff's arrays, this file's own writer and the NumPy
oracle; the availability path reading GeoTIFF paths without rasterio."""

import os
import struct
import zlib

import numpy as np
import pytest

import atlite_b200 as ab
import geotiff_oracle as GO
from atlite_b200 import geotiff, gis
from atlite_b200.engine import GeoTiffOp

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "geotiff")
FIXTURES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.endswith(".tif"))


def _ref(name):
    with np.load(os.path.join(HERE, "golden", "reference_geotiff.npz")) as z:
        return z[name]


# ---------------------------------------------------------------- a GeoTIFF writer for the tests
def lzw_encode(data):
    """TIFF LZW as libtiff writes it: Clear first, MSB-first codes, the width growing one code
    early, Clear when the next free code reaches 4094, EOI last."""
    out, acc, nacc = bytearray(), 0, 0

    def put(code, width):
        nonlocal acc, nacc
        acc = (acc << width) | code
        nacc += width
        while nacc >= 8:
            nacc -= 8
            out.append((acc >> nacc) & 0xFF)
        acc &= (1 << nacc) - 1

    width, nxt, table = 9, 258, {}
    put(256, width)
    if len(data):
        prefix = data[0]
        for b in data[1:]:
            c = table.get((prefix, b))
            if c is not None:
                prefix = c
                continue
            put(prefix, width)
            table[(prefix, b)] = nxt
            nxt += 1
            if nxt == 4094:
                put(256, width)
                table, nxt, width = {}, 258, 9
            elif nxt > (1 << width) - 1:
                width += 1
            prefix = b
        put(prefix, width)
        nxt += 1
        if nxt == 4094:
            put(256, width)
            width = 9
        elif nxt > (1 << width) - 1:
            width += 1
    put(257, width)
    if nacc:
        out.append((acc << (8 - nacc)) & 0xFF)
    return bytes(out)


def _predict(block, predictor, bo):
    """File bytes of one (rows, cols) segment of native samples, predictor applied."""
    dt = block.dtype
    if predictor == 3:
        b = block.astype(dt.newbyteorder(">")).view(np.uint8).reshape(block.shape[0], block.shape[1], dt.itemsize)
        b = np.ascontiguousarray(b.transpose(0, 2, 1)).reshape(block.shape[0], -1)  # planes, MSB first
        b = np.diff(b, axis=1, prepend=np.zeros((b.shape[0], 1), np.uint8)).astype(np.uint8)
        return b.tobytes()
    if predictor == 2:
        u = block.view(np.dtype(f"u{dt.itemsize}"))
        block = np.diff(u, axis=1, prepend=np.zeros((u.shape[0], 1), u.dtype)).astype(u.dtype).view(dt)
    return block.astype(dt.newbyteorder(bo)).tobytes()


def write_tiff(path, arr, *, tiled=False, block=(8, 0), compression=5, predictor=1, bo="<", bigtiff=False,
               epsg=3035, geographic=False, point=False, scale=100.0, origin=(4.0e6, 3.1e6), nodata=None,
               transform=None, override=None, extra=()):
    """Write ``arr`` as a single-band GeoTIFF: ``block`` = (rows, cols) of a tile, or (rows per
    strip, ignored) for strips.  ``override`` {segment: bytes} replaces stored segments (corrupt
    input); ``extra`` adds (tag, type, values) entries."""
    ny, nx = arr.shape
    dt = arr.dtype
    bh, bw = block if tiled else (block[0], nx)
    segs = []
    for r in range(0, ny, bh):
        for c in range(0, nx, bw):
            b = arr[r:r + bh, c:c + bw]
            if tiled and b.shape != (bh, bw):
                pad = np.zeros((bh, bw), dt)
                pad[:b.shape[0], :b.shape[1]] = b
                b = pad
            raw = _predict(np.ascontiguousarray(b), predictor, bo)
            segs.append(lzw_encode(raw) if compression == 5 else zlib.compress(raw) if compression == 8 else raw)
    for k, v in (override or {}).items():
        segs[k] = v
    head = 16 if bigtiff else 8
    offs, pos = [], head
    for s in segs:
        offs.append(pos)
        pos += len(s)
    kind = {"u": 1, "i": 2, "f": 3}[dt.kind]
    long_t = 16 if bigtiff else 4
    tags = [(256, 4, [nx]), (257, 4, [ny]), (258, 3, [8 * dt.itemsize]), (259, 3, [compression]), (262, 3, [1]),
            (277, 3, [1]), (284, 3, [1]), (317, 3, [predictor]), (339, 3, [kind])]
    if tiled:
        tags += [(322, 3, [bw]), (323, 3, [bh]), (324, long_t, offs), (325, long_t, [len(s) for s in segs])]
    else:
        tags += [(273, long_t, offs), (278, 4, [bh]), (279, long_t, [len(s) for s in segs])]
    if transform is not None:
        tags.append((34264, 12, list(transform)))
    else:
        tags += [(33550, 12, [scale, scale, 0.0]), (33922, 12, [0.0, 0.0, 0.0, origin[0], origin[1], 0.0])]
    keys = [(1024, 2 if geographic else 1), (1025, 2 if point else 1)]
    if epsg is not None:
        keys.append((2048 if geographic else 3072, epsg))
    tags.append((34735, 3, [1, 1, 0, len(keys)] + [v for k, x in keys for v in (k, 0, 1, x)]))
    if nodata is not None:
        tags.append((42113, 2, nodata.encode() + b"\0"))
    tags = sorted(tags + list(extra), key=lambda t: t[0])
    fmt = {2: "s", 3: "H", 4: "I", 12: "d", 16: "Q"}
    size = {2: 1, 3: 2, 4: 4, 12: 8, 16: 8}
    ent, inline = (20, 8) if bigtiff else (12, 4)
    ifd_at = pos + (pos & 1)
    data_at = ifd_at + (8 if bigtiff else 2) + len(tags) * ent + (8 if bigtiff else 4)
    entries, blobs = b"", b""
    for tag, typ, vals in tags:
        n = len(vals)
        body = bytes(vals) if typ == 2 else struct.pack(bo + fmt[typ] * n, *vals)
        e = struct.pack(bo + ("HHQ" if bigtiff else "HHI"), tag, typ, n)
        if len(body) <= inline:
            e += body.ljust(inline, b"\0")
        else:
            e += struct.pack(bo + ("Q" if bigtiff else "I"), data_at + len(blobs))
            blobs += body + (b"\0" if len(body) & 1 else b"")
        entries += e
    ifd = struct.pack(bo + ("Q" if bigtiff else "H"), len(tags)) + entries + b"\0" * (8 if bigtiff else 4)
    if bigtiff:
        header = (b"II" if bo == "<" else b"MM") + struct.pack(bo + "HHHQ", 43, 8, 0, ifd_at)
    else:
        header = (b"II" if bo == "<" else b"MM") + struct.pack(bo + "HI", 42, ifd_at)
    with open(path, "wb") as fh:
        fh.write(header + b"".join(segs) + b"\0" * (ifd_at - pos) + ifd + blobs)
    return path


def _content(rng, shape, dt, kind):
    """A constant, a blocky class map, or random bits."""
    if kind == "constant":
        v = np.frombuffer(rng.bytes(dt.itemsize), dtype=dt)[0]
        return np.full(shape, 0 if dt.kind == "f" and not np.isfinite(v) else v, dtype=dt)
    if kind == "blocky":
        c = rng.integers(0, 40, (-(-shape[0] // 5), -(-shape[1] // 5)))
        return np.repeat(np.repeat(c, 5, 0), 5, 1)[:shape[0], :shape[1]].astype(dt)
    return np.frombuffer(rng.bytes(shape[0] * shape[1] * dt.itemsize), dtype=dt).reshape(shape).copy()


DTYPES = ["u1", "i1", "u2", "i2", "u4", "i4", "u8", "i8", "f2", "f4", "f8"]


def _cases(dt):
    """(layout kwargs, compression, predictor, content) for one dtype: every compression, every
    valid predictor, striped (1-row, ~8 KB and odd strips) and tiled (edge tiles) layouts."""
    dt = np.dtype(dt)
    rows_8k = max(1, 8192 // (67 * dt.itemsize))
    layouts = [dict(tiled=False, block=(1, 0)), dict(tiled=False, block=(rows_8k, 0)),
               dict(tiled=False, block=(7, 0)), dict(tiled=True, block=(16, 32)),
               dict(tiled=True, block=(32, 16), bigtiff=True)]
    preds = [1, 2, 3] if dt.kind == "f" else [1, 2]
    kinds = ["constant", "blocky", "random"]
    out, k = [], 0
    for lay in layouts:
        for comp in (1, 5, 8):
            for p in preds if comp != 1 else [1]:  # libtiff ignores a predictor on uncompressed data
                out.append((lay, comp, p, kinds[k % 3]))
                k += 1
    return out


# ---------------------------------------------------------------- CPU
def _golden_cases():
    """{name: case} of tests/golden/make_golden_geotiff.py, what the fixtures were written from."""
    import importlib.util

    spec = importlib.util.spec_from_file_location("make_golden_geotiff",
                                                  os.path.join(HERE, "golden", "make_golden_geotiff.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return {c[0]: c[1:] for c in mod.cases()}


def test_fixture_list_is_complete():
    assert sorted(_golden_cases()) == FIXTURES


@pytest.mark.parametrize("name", FIXTURES)
def test_info_on_libtiff_fixtures(name):
    arr, comp, pred, rps, (epsg, geographic, point), scale, (x0, y0), nodata = _golden_cases()[name]
    inf = geotiff.info(os.path.join(GOLDEN, name + ".tif"))
    block = (min(rps, arr.shape[0]), arr.shape[1])
    assert (inf.shape, inf.dtype, inf.block, inf.predictor) == (arr.shape, arr.dtype, block, pred)
    assert inf.compression == {"tiff_lzw": 5, "tiff_adobe_deflate": 8, "raw": 1}[comp]
    assert inf.epsg == (None if epsg == 32767 else epsg)
    assert inf.byteorder == "<" and not inf.bigtiff and not inf.tiled
    if nodata is None:
        assert inf.nodata is None
    else:
        assert np.array_equal(inf.nodata, float(nodata), equal_nan=True)
    n = -(-arr.shape[0] // block[0])
    assert len(inf.offsets) == len(inf.byte_counts) == n and (np.diff(inf.offsets) > 0).all()
    assert inf.offsets[-1] + inf.byte_counts[-1] <= os.path.getsize(inf.path)
    if point:  # PixelIsPoint: the corner is half a pixel up and left of the tie point
        x0, y0 = x0 - scale / 2, y0 + scale / 2
    assert inf.transform == (scale, 0.0, x0, 0.0, -scale, y0)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_libtiff(name):
    assert np.array_equal(GO.decode(geotiff.info(os.path.join(GOLDEN, name + ".tif"))), _ref(name), equal_nan=True)


def test_writer_files_parse(tmp_path):
    rng = np.random.default_rng(0)
    arr = _content(rng, (45, 67), np.dtype("i2"), "blocky")
    for bo in "<>":
        for big in (False, True):
            p = write_tiff(tmp_path / f"t{bo == '>'}{big}.tif", arr, tiled=True, block=(16, 32), bo=bo, bigtiff=big,
                           predictor=2, epsg=4326, geographic=True, scale=0.5, origin=(1.0, 2.0), nodata="-1")
            inf = geotiff.info(p)
            assert (inf.byteorder, inf.bigtiff, inf.tiled, inf.block, inf.grid) == (bo, big, True, (16, 32), (3, 3))
            assert inf.dtype == np.dtype("int16") and inf.epsg == 4326 and inf.nodata == -1.0
            assert inf.transform == (0.5, 0.0, 1.0, 0.0, -0.5, 2.0)
            assert np.array_equal(GO.decode(inf), arr)
    p = write_tiff(tmp_path / "mt.tif", arr, transform=[2.0, 0, 0, 10.0, 0, -3.0, 0, 20.0] + [0] * 7 + [1])
    assert geotiff.info(p).transform == (2.0, 0.0, 10.0, 0.0, -3.0, 20.0)


def test_writer_agrees_with_libtiff(tmp_path):
    """libtiff decodes this file's writer (tiled, BigTIFF, big-endian, LZW with Clears) to the
    source arrays, so the writer and the decoder cannot share a mistake."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(1)
    n = 0
    for dt in ("u1", "u2", "i2", "i4", "f4", "f8"):
        for kind in ("blocky", "random"):
            arr = _content(rng, (45, 67), np.dtype(dt), kind)
            for lay, comp, p, _ in _cases(dt)[::2]:
                for bo in "<>":
                    path = write_tiff(tmp_path / f"w{n}.tif", arr, compression=comp, predictor=p, bo=bo, **lay)
                    back = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
                    assert back is not None, (dt, lay, comp, p, bo)
                    assert np.array_equal(back.view(np.dtype(dt).newbyteorder("=")), arr, equal_nan=True), (
                        dt, kind, lay, comp, p, bo)
                    n += 1
    assert n > 100


def test_window_arithmetic(tmp_path):
    p = write_tiff(tmp_path / "w.tif", np.zeros((50, 80), np.uint8), scale=10.0, origin=(1000.0, 2000.0))
    inf = geotiff.info(p)
    assert geotiff.window(inf, None) == ((0, 50), (0, 80))
    assert geotiff.window(inf, (1000.0, 1500.0, 1800.0, 2000.0)) == ((0, 50), (0, 80))
    assert geotiff.window(inf, (900.0, 1400.0, 1900.0, 2100.0)) == ((0, 50), (0, 80))  # clipped
    assert geotiff.window(inf, (1015.0, 1905.0, 1035.0, 1995.0)) == ((0, 10), (1, 4))
    assert geotiff.window(inf, (1020.0, 1900.0, 1030.0, 1990.0)) == ((1, 10), (2, 3))  # exact edges: no sliver
    assert geotiff.window(inf, (1020.0 + 1e-12, 1900.0, 1030.0 - 1e-12, 1990.0)) == ((1, 10), (2, 3))
    with pytest.raises(ValueError, match="do not overlap"):
        geotiff.window(inf, (0.0, 0.0, 999.0, 100.0))
    with pytest.raises(ValueError, match="do not overlap"):
        geotiff.window(inf, (1800.0, 1500.0, 1900.0, 2000.0))
    assert list(inf.segments_in(0, 8, 0, 80)) == [0] and list(inf.segments_in(7, 9, 5, 6)) == [0, 1]
    t = geotiff.info(write_tiff(tmp_path / "t.tif", np.zeros((50, 80), np.uint8), tiled=True, block=(16, 32)))
    assert list(t.segments_in(15, 17, 31, 33)) == [0, 1, 3, 4] and list(t.segments_in(48, 50, 64, 80)) == [11]


def test_refused_layouts(tmp_path):
    arr = np.zeros((20, 30), np.uint8)
    p = write_tiff(tmp_path / "a.tif", arr, compression=7)
    with pytest.raises(NotImplementedError, match="tag 259 = 7"):
        geotiff.info(p)
    for comp in (32773, 50000, 34887):  # PackBits, ZSTD, LERC
        with pytest.raises(NotImplementedError, match=f"259 = {comp}"):
            geotiff.info(_retag(write_tiff(tmp_path / f"c{comp}.tif", arr, compression=1), 259, comp))
    with pytest.raises(NotImplementedError, match="tag 277 = 3"):
        geotiff.info(_retag(write_tiff(tmp_path / "s.tif", arr, compression=1), 277, 3))
    for bits in (1, 4, 12):
        with pytest.raises(NotImplementedError, match="tag 258"):
            geotiff.info(_retag(write_tiff(tmp_path / f"b{bits}.tif", arr, compression=1), 258, bits))
    with pytest.raises(NotImplementedError, match="tag 339 = 4"):
        geotiff.info(_retag(write_tiff(tmp_path / "f.tif", arr, compression=1), 339, 4))
    with pytest.raises(NotImplementedError, match="tag 317 = 3"):
        geotiff.info(write_tiff(tmp_path / "p3.tif", arr, predictor=3))
    with pytest.raises(NotImplementedError, match="tag 317 = 34892"):
        geotiff.info(_retag(write_tiff(tmp_path / "p.tif", arr, compression=8), 317, 34892))
    assert geotiff.info(write_tiff(tmp_path / "p1.tif", arr, compression=1, predictor=3)).predictor == 1
    with pytest.raises(NotImplementedError, match="tag 34264"):
        geotiff.info(write_tiff(tmp_path / "r.tif", arr, transform=[1.0, 0.5, 0, 0, 0.0, -1.0, 0, 0] + [0] * 7 + [1]))
    with pytest.raises(ValueError, match="not a TIFF"):
        geotiff.info(os.path.join(HERE, "golden", "reference_geotiff.npz"))
    assert not geotiff.is_tiff(os.path.join(HERE, "golden", "reference_geotiff.npz"))
    assert not geotiff.is_tiff(tmp_path / "missing.tif") and geotiff.is_tiff(p)


def _retag(path, tag, value):
    """Rewrite the first short value of ``tag`` in a little-endian classic TIFF."""
    b = bytearray(open(path, "rb").read())
    ifd = struct.unpack("<I", b[4:8])[0]
    n = struct.unpack("<H", b[ifd:ifd + 2])[0]
    for k in range(n):
        e = ifd + 2 + 12 * k
        if struct.unpack("<H", b[e:e + 2])[0] == tag:
            b[e + 8:e + 12] = struct.pack("<I", value) if struct.unpack("<H", b[e + 2:e + 4])[0] == 4 else \
                struct.pack("<HH", value, 0)
            break
    else:
        raise KeyError(tag)
    open(path, "wb").write(bytes(b))
    return path


def test_missing_crs(tmp_path):
    p = write_tiff(tmp_path / "n.tif", np.zeros((20, 30), np.uint8), epsg=None)
    assert geotiff.info(p).epsg is None
    with pytest.raises(ValueError, match=r"please provide it manually \(crs=\)"):
        geotiff.read(p)
    u = os.path.join(GOLDEN, "lc_u8_lzw_p2_userdefined.tif")
    with pytest.raises(ValueError, match=r"please provide it manually \(crs=\)"):
        geotiff.read(u)
    assert not geotiff.readable(u) and geotiff.readable(u, crs=3035) and geotiff.readable(p, 3035)
    assert not geotiff.readable(tmp_path / "missing.tif", 3035)


# ---------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures_bitwise_libtiff(name):
    r = gis.read_raster(os.path.join(GOLDEN, name + ".tif"), crs=3035)
    got = r.array.cpu().numpy()
    want = _ref(name)
    assert r.array.is_cuda and got.dtype == want.dtype
    assert np.array_equal(got.view(f"u{got.itemsize}"), want.view(f"u{want.itemsize}"))
    inf = geotiff.info(os.path.join(GOLDEN, name + ".tif"))
    assert r.transform == inf.transform and r.epsg == (inf.epsg or 3035)
    assert (r.nodata is None and inf.nodata is None) or np.array_equal(r.nodata, inf.nodata, equal_nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("bo", ["<", ">"])
def test_random_rasters_bitwise(tmp_path, dt, bo):
    rng = np.random.default_rng(DTYPES.index(dt) * 2 + (bo == ">"))
    for n, (lay, comp, p, kind) in enumerate(_cases(dt)):
        arr = _content(rng, (45, 67), np.dtype(dt), kind)
        path = write_tiff(tmp_path / f"r{n}.tif", arr, compression=comp, predictor=p, bo=bo, **lay)
        got = geotiff.read(path).array.cpu().numpy()
        assert np.array_equal(got.view(f"u{arr.itemsize}"), arr.view(f"u{arr.itemsize}")), (dt, bo, lay, comp, p, kind)


@pytest.mark.gpu
def test_random_bytes_reach_the_12_bit_limit(tmp_path):
    rng = np.random.default_rng(5)
    arr = _content(rng, (301, 257), np.dtype("u1"), "random")
    assert len(lzw_encode(arr[:100].tobytes())) > 100 * 257  # incompressible: the table fills several times
    for lay in (dict(tiled=False, block=(100, 0)), dict(tiled=True, block=(128, 128))):
        p = write_tiff(tmp_path / "big.tif", arr, **lay)
        assert np.array_equal(geotiff.read(p).array.cpu().numpy(), arr)


@pytest.mark.gpu
@pytest.mark.parametrize("tiled", [False, True])
def test_windows_read_only_their_segments(tmp_path, tiled):
    rng = np.random.default_rng(2)
    arr = _content(rng, (203, 157), np.dtype("f4"), "blocky") + rng.normal(0, 1, (203, 157)).astype(np.float32)
    p = write_tiff(tmp_path / "w.tif", arr, tiled=tiled, block=(32, 48) if tiled else (9, 0), predictor=3,
                   epsg=4326, geographic=True, scale=0.5, origin=(10.0, 60.0))
    inf = geotiff.info(p)
    whole = geotiff.read(p).array.cpu().numpy()
    assert np.array_equal(whole, arr)
    a, _, c, _, e, f = inf.transform
    for r0, r1, c0, c1 in [(0, 203, 0, 157), (0, 5, 0, 157), (198, 203, 100, 157), (50, 60, 0, 3), (40, 41, 150, 157),
                           (33, 60, 50, 90), (10, 190, 5, 150), (96, 100, 96, 100)]:
        bounds = (c + c0 * a, f + r1 * e, c + c1 * a, f + r0 * e)
        r = geotiff.read(p, bounds)
        assert np.array_equal(r.array.cpu().numpy(), whole[r0:r1, c0:c1]), (r0, r1, c0, c1)
        assert r.transform == (a, 0.0, c + c0 * a, 0.0, e, f + r0 * e)
        op = GeoTiffOp()
        got = op(inf, *geotiff.window(inf, bounds))
        assert np.array_equal(got.cpu().numpy(), whole[r0:r1, c0:c1])
        bh, bw = inf.block
        want = (-(-r1 // bh) - r0 // bh) * (-(-c1 // bw) - c0 // bw)
        assert op.stats["segments"] == want, (r0, r1, c0, c1, op.stats)
        assert op.stats["stored_bytes"] == inf.byte_counts[inf.segments_in(r0, r1, c0, c1)].sum()


@pytest.mark.gpu
@pytest.mark.parametrize("comp", [1, 5, 8])
def test_batch_sizes_give_the_same_bits(tmp_path, comp):
    rng = np.random.default_rng(3)
    arr = _content(rng, (190, 170), np.dtype("u2"), "blocky") + rng.integers(0, 3, (190, 170)).astype(np.uint16)
    p = write_tiff(tmp_path / "b.tif", arr, tiled=True, block=(16, 32), compression=comp,
                   predictor=1 if comp == 1 else 2, bo=">")
    inf = geotiff.info(p)
    batches = []
    for bb in (1, 700, 5000, 40000, 64 << 20):
        op = GeoTiffOp(batch_bytes=bb, n_threads=3)
        got = op(inf, (0, 190), (0, 170)).cpu().numpy()
        assert np.array_equal(got, arr), bb
        batches.append(op.stats["batches"])
    assert batches[0] == len(inf.offsets) and batches[-1] == 1 and batches == sorted(batches, reverse=True)


@pytest.mark.gpu
def test_corrupt_segments_raise(tmp_path):
    arr = _content(np.random.default_rng(4), (40, 64), np.dtype("u1"), "blocky")
    good = lzw_encode(arr[16:32, :32].tobytes())

    def codes(*cs):  # 9-bit codes, MSB-first
        bits = "".join(format(c, "09b") for c in cs)
        bits += "0" * (-len(bits) % 8)
        return bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))

    too_long = lzw_encode(np.tile(arr[16:32, :32].ravel(), 2)[:16 * 32 + 40].tobytes())
    cases = {"truncated": good[:len(good) // 2], "past the end of the string table": codes(256, 65, 259, 257),
             "more bytes": too_long, "old-style": b"\x00\x01" + good[2:],
             "end-of-information": codes(256, 65, 66, 257)}
    for reason, seg in cases.items():
        p = write_tiff(tmp_path / "c.tif", arr, tiled=True, block=(16, 32), override={2: seg})
        with pytest.raises(ValueError, match=f"segment 2: .*{reason}"):
            geotiff.read(p)
        op = GeoTiffOp()  # the other segments still decode
        inf = geotiff.info(p)
        assert np.array_equal(op(inf, (0, 16), (0, 64)).cpu().numpy(), arr[:16])
    p = write_tiff(tmp_path / "d.tif", arr, compression=8, override={1: b"not zlib"})
    with pytest.raises(ValueError, match="segment 1: Deflate"):
        geotiff.read(p)


def _landcover(tmp_path, res=1000.0):
    from atlite_b200 import proj

    lon, lat = np.meshgrid(np.linspace(-5.0, 2.5, 30), np.linspace(55.0, 62.0, 30))
    x, y = proj.laea_forward(lon.ravel(), lat.ravel())
    x0, y1 = np.floor(x.min() / res) * res - 5 * res, np.ceil(y.max() / res) * res + 5 * res
    nx, ny = int((x.max() - x0) / res) + 10, int((y1 - y.min()) / res) + 10
    lc = _content(np.random.default_rng(9), (ny, nx), np.dtype("u1"), "blocky")
    path = write_tiff(tmp_path / "landcover.tif", lc, tiled=True, block=(256, 256), predictor=2, scale=res,
                      origin=(x0, y1))
    return path, gis.Raster(lc, (res, 0.0, x0, 0.0, -res, y1), 3035)


@pytest.mark.gpu
def test_availability_with_geotiff_paths(tmp_path):
    from atlite_b200 import synthetic as syn

    X0, Y0, X1, Y1 = -4.0, 56.0, 1.5, 61.0
    cut = ab.Cutout(data=syn.make_dataset(23, 21, 2, x0=X0, y0=Y0, kinds=()))
    shapes = [np.array([[X0 + 1, Y0 + 1], [X1 - 1, Y0 + 1], [X1 - 1, Y1 - 1], [X0 + 1, Y1 - 1]]),
              np.array([[X0 + 0.5, Y0 + 0.5], [X0 + 3, Y0 + 0.7], [X0 + 2, Y0 + 3.5]])]
    path, lc = _landcover(tmp_path)
    rng = np.random.default_rng(10)
    depth = (_content(rng, (300, 400), np.dtype("f4"), "blocky") * -3.0 + rng.normal(0, 1, (300, 400))).astype(
        np.float32)
    dpath = write_tiff(tmp_path / "depth.tif", depth, tiled=True, block=(64, 64), predictor=3, epsg=4326,
                       geographic=True, scale=0.02, origin=(-5.0, 62.0))
    dr = gis.Raster(depth, (0.02, 0.0, -5.0, 0.0, -0.02, 62.0), 4326)
    results = []
    for land, sea in ((str(path), dpath), (lc, dr)):
        ex = gis.ExclusionContainer(3035, 1000)
        ex.add_raster(land, codes=[1, 2, 3, 5, 8, 13, 21, 34], buffer=1500)
        ex.add_raster(sea, codes=lambda d: d < -50.0, nodata=np.nan)
        assert ex.all_closed == isinstance(land, str)
        A = cut.availabilitymatrix(shapes, ex)
        mask, t = ex.compute_shape_availability(shapes[0], crs=4326)
        results.append((np.asarray(A.values), mask, t))
        if isinstance(land, str):
            assert ex.all_open and ex.rasters[0]["raster"].array.is_cuda
    (a1, m1, t1), (a2, m2, t2) = results
    assert np.array_equal(a1, a2) and np.array_equal(m1, m2) and tuple(t1) == tuple(t2)
    assert 0.05 < a1.max() <= 1.0 and m1.any() and not m1.all()


@pytest.mark.gpu
def test_add_raster_path_with_crs_argument(tmp_path):
    """A GeoTIFF whose GeoKeys name no EPSG code takes ``crs=`` when rasterio is not installed."""
    try:
        import rasterio  # noqa: F401
        pytest.skip("with rasterio installed such a file takes the rasterio route")
    except ImportError:
        pass
    arr = _content(np.random.default_rng(11), (50, 60), np.dtype("u1"), "blocky")
    p = write_tiff(tmp_path / "nocrs.tif", arr, epsg=None, scale=100.0, origin=(4.0e6, 3.1e6))
    shape = np.array([[4.0005e6, 3.0955e6], [4.005e6, 3.0955e6], [4.005e6, 3.0995e6]])
    masks = []
    for r in (str(p), gis.Raster(arr, (100.0, 0.0, 4.0e6, 0.0, -100.0, 3.1e6), 3035)):
        ex = gis.ExclusionContainer(3035, 50)
        ex.add_raster(r, codes=[1, 2, 3], crs=3035)
        masks.append(ex.compute_shape_availability(shape, crs=3035)[0])
    assert np.array_equal(*masks)


@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_rasterio_equality(name):
    rasterio = pytest.importorskip("rasterio")
    path = os.path.join(GOLDEN, name + ".tif")
    if geotiff.info(path).epsg is None:
        pytest.skip("no EPSG code: rasterio route")
    with rasterio.open(path) as ds:
        want, t, epsg = ds.read(1), tuple(ds.transform)[:6], ds.crs.to_epsg()
    r = geotiff.read(path)
    assert np.array_equal(r.array.cpu().numpy(), want, equal_nan=True)
    assert r.transform == t and r.epsg == epsg
