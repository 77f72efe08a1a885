"""GeoTIFF rasters without rasterio: ``read`` gives a ``gis.Raster`` whose array is already on the
GPU, for ``ExclusionContainer.add_raster`` (which reads GeoTIFF paths this way).

The first IFD is parsed here (``struct`` over the header, classic TIFF or BigTIFF, ``II`` or
``MM``); overviews are ignored.  The segments (tiles or strips) a window needs are read, decoded
and placed by ``engine.GeoTiffOp`` (csrc/geotiff.cu): LZW and Deflate (csrc/inflate.cu) are
decoded on the GPU from the compressed bytes, uncompressed segments are copied, and one
kernel undoes the predictor and the byte order.  Semantics and what is refused: DESIGN.md
section 1.
"""

from __future__ import annotations

import math
import os
import struct
from dataclasses import dataclass, field

import numpy as np

# TIFF and GeoTIFF tags
WIDTH, HEIGHT, BITS, COMPRESSION = 256, 257, 258, 259
STRIP_OFFSETS, SAMPLES, ROWS_PER_STRIP, STRIP_COUNTS = 273, 277, 278, 279
PLANAR, PREDICTOR = 284, 317
TILE_WIDTH, TILE_LENGTH, TILE_OFFSETS, TILE_COUNTS = 322, 323, 324, 325
SAMPLE_FORMAT = 339
PIXEL_SCALE, TIEPOINT, MODEL_TRANSFORM = 33550, 33922, 34264
GEO_KEYS, GDAL_NODATA = 34735, 42113
# GeoKeys
RASTER_TYPE, GEOGRAPHIC_TYPE, PROJECTED_TYPE = 1025, 2048, 3072
PIXEL_IS_POINT = 2
USER_DEFINED = 32767

COMPRESSIONS = {1: "none", 5: "lzw", 8: "deflate", 32946: "deflate"}
# field type -> (struct code, bytes)
_TYPES = {1: ("B", 1), 2: ("s", 1), 3: ("H", 2), 4: ("I", 4), 5: ("II", 8), 6: ("b", 1), 7: ("B", 1), 8: ("h", 2),
          9: ("i", 4), 10: ("ii", 8), 11: ("f", 4), 12: ("d", 8), 16: ("Q", 8), 17: ("q", 8), 18: ("Q", 8)}


@dataclass
class TiffInfo:
    """What ``info`` reads from a GeoTIFF's first IFD.  ``block`` is (rows, columns) of a tile, or
    (rows per strip, width) for strips; ``dtype`` is native-endian, ``byteorder`` the file's
    (``"<"`` for ``II``, ``">"`` for ``MM``); ``transform`` the north-up (a, b, c, d, e, f) or None;
    ``epsg`` the GeoKeys' EPSG code or None; ``nodata`` the GDAL_NODATA value or None.  ``offsets``
    and ``byte_counts`` are the segment table, row-major."""

    path: str
    shape: tuple
    dtype: np.dtype
    byteorder: str
    bigtiff: bool
    tiled: bool
    block: tuple
    compression: int
    predictor: int
    transform: tuple | None
    epsg: int | None
    nodata: float | None
    offsets: np.ndarray = field(repr=False)
    byte_counts: np.ndarray = field(repr=False)

    @property
    def grid(self):
        """(segments down, segments across)."""
        (ny, nx), (bh, bw) = self.shape, self.block
        return -(-ny // bh), -(-nx // bw)

    def segments_in(self, r0, r1, c0, c1):
        """Row-major numbers of the segments that intersect rows [r0, r1) x columns [c0, c1)."""
        (bh, bw), (_, across) = self.block, self.grid
        rows = np.arange(r0 // bh, (r1 - 1) // bh + 1)
        cols = np.arange(c0 // bw, (c1 - 1) // bw + 1)
        return (rows[:, None] * across + cols[None, :]).ravel()


def _not_supported(tag, value, what):
    return NotImplementedError(f"GeoTIFF tag {tag} = {value!r}: {what} is not supported")


def _read_ifd(fh, path):
    """(byte order, BigTIFF, {tag: value tuple or bytes}) of the first IFD."""
    head = fh.read(16)
    if len(head) < 8 or head[:2] not in (b"II", b"MM"):
        raise ValueError(f"{path} is not a TIFF file")
    bo = "<" if head[:2] == b"II" else ">"
    magic = struct.unpack(bo + "H", head[2:4])[0]
    if magic == 42:
        big, ifd = False, struct.unpack(bo + "I", head[4:8])[0]
    elif magic == 43 and len(head) == 16 and struct.unpack(bo + "HH", head[4:8]) == (8, 0):
        big, ifd = True, struct.unpack(bo + "Q", head[8:16])[0]
    else:
        raise ValueError(f"{path} is not a TIFF file (magic number {magic})")
    cnt_fmt, ent_size, val_size, off_fmt = ("Q", 20, 8, "Q") if big else ("H", 12, 4, "I")  # off_fmt: also counts
    fh.seek(ifd)
    raw = fh.read(struct.calcsize(cnt_fmt))
    if len(raw) < struct.calcsize(cnt_fmt):
        raise ValueError(f"{path}: the first IFD lies past the end of the file")
    n = struct.unpack(bo + cnt_fmt, raw)[0]
    entries = fh.read(n * ent_size)
    if len(entries) < n * ent_size:
        raise ValueError(f"{path}: the first IFD is truncated")
    tags = {}
    for k in range(n):
        e = entries[k * ent_size:(k + 1) * ent_size]
        tag, typ = struct.unpack(bo + "HH", e[:4])
        count = struct.unpack(bo + off_fmt, e[4:4 + val_size])[0]
        if typ not in _TYPES:
            continue  # a type this reader never needs
        code, size = _TYPES[typ]
        nbytes = size * count
        body = e[ent_size - val_size:]
        if nbytes > val_size:
            fh.seek(struct.unpack(bo + off_fmt, body)[0])
            body = fh.read(nbytes)
            if len(body) < nbytes:
                raise ValueError(f"{path}: the value of tag {tag} lies past the end of the file")
        body = body[:nbytes]
        if typ == 2:
            tags[tag] = body
        else:
            tags[tag] = struct.unpack(bo + code[0] * (count * len(code)), body)
    return bo, big, tags


def _geokeys(tags):
    """{GeoKey: value} of the short-valued keys of the GeoKeyDirectory."""
    d = tags.get(GEO_KEYS)
    if not d or len(d) < 4:
        return {}
    keys = {}
    for k in range(min(d[3], (len(d) - 4) // 4)):
        key, loc, count, value = d[4 + 4 * k:8 + 4 * k]
        if loc == 0 and count == 1:
            keys[key] = value
    return keys


def _transform(tags, keys):
    if MODEL_TRANSFORM in tags:
        m = tags[MODEL_TRANSFORM]
        if len(m) != 16:
            raise ValueError(f"ModelTransformationTag needs 16 values, not {len(m)}")
        if m[1] != 0.0 or m[4] != 0.0:
            raise _not_supported(MODEL_TRANSFORM, tuple(m), "a rotated or sheared transform")
        a, c, e, f = m[0], m[3], m[5], m[7]
    elif PIXEL_SCALE in tags and TIEPOINT in tags:
        tp, (sx, sy) = tags[TIEPOINT], tags[PIXEL_SCALE][:2]
        if len(tp) != 6:
            raise _not_supported(TIEPOINT, tuple(tp), f"{len(tp) // 6} tie points (a warped raster)")
        i, j, _, x, y, _ = tp
        a, c, e, f = sx, x - i * sx, -sy, y + j * sy
    else:
        return None
    if keys.get(RASTER_TYPE) == PIXEL_IS_POINT:  # the corner is half a pixel up and left
        c, f = c - a / 2, f - e / 2
    return (float(a), 0.0, float(c), 0.0, float(e), float(f))


def info(path):
    """A ``TiffInfo`` of the GeoTIFF at ``path``.  Raises ``ValueError`` for a file that is not a
    well-formed TIFF and ``NotImplementedError``, naming the tag and its value, for a layout the
    reader does not support (see DESIGN.md section 1)."""
    path = os.fspath(path)
    with open(path, "rb") as fh:
        bo, big, tags = _read_ifd(fh, path)

    def one(tag, default=None):
        v = tags.get(tag)
        if v is None:
            if default is None:
                raise ValueError(f"{path}: required TIFF tag {tag} is missing")
            return default
        return v[0]

    nx, ny = one(WIDTH), one(HEIGHT)
    spp = one(SAMPLES, 1)
    if spp != 1:
        raise _not_supported(SAMPLES, spp, "more than one sample per pixel")
    bits = tags.get(BITS, (1,))
    if len(set(bits)) != 1 or bits[0] not in (8, 16, 32, 64):
        raise _not_supported(BITS, tuple(bits), f"{bits[0]}-bit samples")
    bits = bits[0]
    fmt = tags.get(SAMPLE_FORMAT, (1,))[0]
    kind = {1: "u", 2: "i", 3: "f"}.get(fmt)
    if kind is None:
        raise _not_supported(SAMPLE_FORMAT, fmt, "this sample format")
    try:
        dtype = np.dtype(f"{kind}{bits // 8}")
    except TypeError:
        raise _not_supported(BITS, bits, f"{bits}-bit {'float' if kind == 'f' else 'integer'} samples") from None
    comp = one(COMPRESSION, 1)
    if comp not in COMPRESSIONS:
        raise _not_supported(COMPRESSION, comp, "this compression (only none 1, LZW 5 and Deflate 8 / 32946 are)")
    pred = one(PREDICTOR, 1) if comp != 1 else 1  # libtiff applies no predictor to uncompressed data
    if pred not in (1, 2, 3) or (pred == 3 and kind != "f"):
        raise _not_supported(PREDICTOR, pred, f"predictor {pred} for {dtype} samples")
    if TILE_WIDTH in tags or TILE_OFFSETS in tags:
        tiled, block = True, (one(TILE_LENGTH), one(TILE_WIDTH))
        offsets, counts = tags.get(TILE_OFFSETS), tags.get(TILE_COUNTS)
    else:
        rps = one(ROWS_PER_STRIP, 2 ** 32 - 1)
        tiled, block = False, (max(1, min(rps, ny)), nx)
        offsets, counts = tags.get(STRIP_OFFSETS), tags.get(STRIP_COUNTS)
    if nx <= 0 or ny <= 0 or block[0] <= 0 or block[1] <= 0:
        raise ValueError(f"{path}: empty image or segment ({ny} x {nx}, segments {block})")
    n_seg = -(-ny // block[0]) * -(-nx // block[1])
    if offsets is None or counts is None or len(offsets) < n_seg or len(counts) < n_seg:
        raise ValueError(f"{path}: the segment table has fewer than the {n_seg} segments of the image")
    keys = _geokeys(tags)
    epsg = keys.get(PROJECTED_TYPE) or keys.get(GEOGRAPHIC_TYPE)
    if epsg is not None and not 0 < epsg < USER_DEFINED:
        epsg = None
    nodata = None
    if GDAL_NODATA in tags:
        txt = tags[GDAL_NODATA].split(b"\0")[0].decode("ascii", "replace").strip()
        try:
            nodata = float(txt)
        except ValueError:
            raise ValueError(f"{path}: GDAL_NODATA {txt!r} is not a number") from None
    return TiffInfo(path=path, shape=(int(ny), int(nx)), dtype=dtype, byteorder=bo, bigtiff=big, tiled=tiled,
                    block=(int(block[0]), int(block[1])), compression=int(comp), predictor=int(pred),
                    transform=_transform(tags, keys), epsg=epsg, nodata=nodata,
                    offsets=np.asarray(offsets[:n_seg], dtype=np.int64),
                    byte_counts=np.asarray(counts[:n_seg], dtype=np.int64))


def is_tiff(path):
    """Does ``path`` name a file that starts with a TIFF or BigTIFF header?"""
    try:
        with open(path, "rb") as fh:
            head = fh.read(4)
    except (OSError, TypeError):
        return False
    return head in (b"II*\0", b"MM\0*", b"II+\0", b"MM\0+")


def window(inf, bounds):
    """((r0, r1), (c0, c1)): the rows and columns of every pixel ``bounds`` = (left, bottom, right,
    top) overlap by more than ``gis.REGRID_EPS`` pixel, clipped to the raster (``gebco.raster``'s
    rule); None: the whole raster.  Bounds that do not overlap raise ``ValueError``."""
    from .gebco import window as from_bounds
    from .gis import REGRID_EPS

    ny, nx = inf.shape
    if bounds is None:
        return (0, ny), (0, nx)
    col_off, row_off, width, height = from_bounds(_north_up(inf), *(float(b) for b in bounds))
    c0, c1 = max(0, math.floor(col_off + REGRID_EPS)), min(nx, math.ceil(col_off + width - REGRID_EPS))
    r0, r1 = max(0, math.floor(row_off + REGRID_EPS)), min(ny, math.ceil(row_off + height - REGRID_EPS))
    if c1 <= c0 or r1 <= r0:
        raise ValueError(f"bounds {tuple(bounds)} do not overlap the raster {inf.path}")
    return (r0, r1), (c0, c1)


def _north_up(inf):
    if inf.transform is None:
        raise ValueError(f"{inf.path} has no georeferencing (ModelPixelScale + ModelTiepoint or "
                         "ModelTransformation)")
    a, b, _, d, e, _ = inf.transform
    if b != 0.0 or d != 0.0 or not a > 0.0 or not e < 0.0:
        raise ValueError("only north-up rasters are supported (transform b = d = 0, a > 0, e < 0)")
    return inf.transform


def read(path, bounds=None, crs=None, device=None):
    """The GeoTIFF at ``path`` as ``gis.Raster(array, transform, crs)`` with ``array`` a (ny, nx)
    CUDA tensor of the file's dtype on ``device`` (default: the current one), and ``nodata`` the
    file's GDAL_NODATA (or None).  ``bounds`` = (left, bottom, right, top) in the raster's CRS
    reads only the window ``window`` gives, and only the segments that intersect it; the transform
    is the window's.  The CRS is the GeoKeys' EPSG code, else ``crs``, else ``ValueError``."""
    from . import proj
    from .engine import GeoTiffOp
    from .gis import Raster

    inf = info(path)
    a, _, c, _, e, f = _north_up(inf)
    src = inf.epsg if inf.epsg is not None else crs
    if src is None:
        raise ValueError(f"CRS of {inf.path} is undefined, please provide it manually (crs=)")
    proj.epsg(src)  # an unsupported CRS fails before any device work
    (r0, r1), (c0, c1) = window(inf, bounds)
    array = GeoTiffOp(device)(inf, (r0, r1), (c0, c1))
    return Raster(array, (a, 0.0, c + c0 * a, 0.0, e, f + r0 * e), src, nodata=inf.nodata)


def readable(path, crs=None):
    """Can ``read`` open ``path`` without a ``crs`` it lacks?  True for an existing file with a TIFF
    or BigTIFF header, a layout ``info`` accepts, a north-up georeferencing and a CRS that resolves:
    the GeoKeys name an EPSG code, or ``crs`` is given."""
    if not is_tiff(path):
        return False
    try:
        inf = info(path)
        _north_up(inf)
    except (NotImplementedError, ValueError, OSError):
        return False
    return inf.epsg is not None or crs is not None
