"""GeoTIFF band decode restated in NumPy and plain Python (csrc/geotiff.cu's semantics).

``decode(info)`` takes the segment table ``atlite_b200.geotiff.info`` parsed and returns the whole
band as a native-endian NumPy array: each segment is read, LZW-decoded code by code with a table
of byte strings (or inflated with zlib, or taken as it is), the predictor undone row by row, and
its pixels copied into the image, edge tiles clipped.  Slow, and meant for small files.
"""

import zlib

import numpy as np


def lzw_decode(data, size):
    """The ``size`` bytes a TIFF LZW segment decodes to (MSB-first codes, Clear 256, EOI 257, widths
    9 to 12 bits, changing one code early); raises ValueError for a corrupt segment."""
    if len(data) >= 2 and data[0] == 0 and data[1] & 1:
        raise ValueError("old-style LZW")
    bits = np.unpackbits(np.frombuffer(bytes(data), dtype=np.uint8))
    out = bytearray()
    table, prev, pos, width = None, None, 0, 9

    def reset():
        return [bytes([i]) for i in range(256)] + [b"", b""]

    table = reset()
    while True:
        if pos + width > len(bits):
            if len(out) == size:
                return bytes(out)
            raise ValueError("truncated")
        code = int("".join("1" if b else "0" for b in bits[pos:pos + width]), 2)
        pos += width
        if code == 257:
            if len(out) != size:
                raise ValueError("short")
            return bytes(out)
        if code == 256:
            table, prev, width = reset(), None, 9
            continue
        if len(out) == size:
            raise ValueError("long")
        if code < len(table):
            s = table[code]
        elif code == len(table) and prev is not None:
            s = prev + prev[:1]
        else:
            raise ValueError("bad code")
        out += s
        if len(out) > size:
            raise ValueError("long")
        if prev is not None and len(table) < 4096:
            table.append(prev + s[:1])
            n = len(table)
            width = 9 if n < 511 else 10 if n < 1023 else 11 if n < 2047 else 12
        prev = s


def _unpredict(raw, rows, cols, dtype, byteorder, predictor):
    """(rows, cols) native samples of one decoded segment."""
    nb = dtype.itemsize
    if predictor == 3:  # byte running sum over the row, then planes most significant first
        b = np.frombuffer(raw, dtype=np.uint8).reshape(rows, cols * nb)
        b = np.cumsum(b, axis=1, dtype=np.uint64).astype(np.uint8)
        planes = b.reshape(rows, nb, cols).transpose(0, 2, 1)  # (row, col, byte from the most significant)
        return np.ascontiguousarray(planes).view(dtype.newbyteorder(">")).reshape(rows, cols).astype(dtype)
    a = np.frombuffer(raw, dtype=dtype.newbyteorder(byteorder)).reshape(rows, cols).astype(dtype)
    if predictor == 2:
        u = a.view(np.dtype(f"u{nb}"))
        a = np.cumsum(u, axis=1, dtype=np.uint64).astype(u.dtype).view(dtype)
    return a


def decode(info):
    """The whole band of the file ``info`` describes, as a (ny, nx) native NumPy array."""
    ny, nx = info.shape
    bh, bw = info.block
    down, across = info.grid
    out = np.empty((ny, nx), dtype=info.dtype)
    with open(info.path, "rb") as fh:
        for k in range(down * across):
            r0, c0 = (k // across) * bh, (k % across) * bw
            rows = bh if info.tiled else min(bh, ny - r0)
            size = rows * bw * info.dtype.itemsize
            fh.seek(int(info.offsets[k]))
            data = fh.read(int(info.byte_counts[k]))
            if info.compression == 5:
                raw = lzw_decode(data, size)
            elif info.compression in (8, 32946):
                raw = zlib.decompress(data)
            else:
                raw = data[:size]
            if len(raw) != size:
                raise ValueError(f"segment {k} decodes to {len(raw)} bytes, not {size}")
            seg = _unpredict(raw, rows, bw, info.dtype, info.byteorder, info.predictor)
            h, w = min(rows, ny - r0), min(bw, nx - c0)
            out[r0:r0 + h, c0:c0 + w] = seg[:h, :w]
    return out
