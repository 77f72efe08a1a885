"""Time geotiff.read on the land-cover raster of tools/prof_availability.py: 40000 x 40000 uint8
pixels (1.6e9, EPSG:3035 at 100 m), as a tiled LZW GeoTIFF (256 x 256 tiles) and as a striped one
(1-row strips, GDAL's layout for rows above 8 KB).

Pure-Python LZW is far too slow for 1.6e9 pixels, so ``--pool`` realistic segments (class maps of
44 codes in 2 km patches, as prof_availability draws them) are encoded once and the file is
assembled from them in a random arrangement: the decode work per segment is realistic and the
expected array is known.  Reported per layout: reading the compressed bytes (page cache), their
host -> device copy from pinned memory, the decode and placement kernels (torch.profiler, a run of
their own), geotiff.read's wall time (best of --repeat), and for comparison today's cost of a
decoded array, ``torch.from_numpy(decoded).to("cuda")`` from pageable memory; then
prof_availability's availabilitymatrix with the land cover given as the tiled GeoTIFF path against
the same array given as a gis.Raster (equal results asserted).  Files go to a temporary directory.

    python tools/prof_geotiff.py [--pool 48] [--repeat 3] [--regions 300] [--out PATH]
"""

import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from atlite_b200 import geotiff, gis  # noqa: E402
from test_geotiff import lzw_encode  # noqa: E402

N, RES, X0, Y0 = 40000, 100.0, 2.0e6, 1.0e6


def class_map(rng, shape, patch=20):
    coarse = rng.integers(0, 44, (-(-shape[0] // patch) + 1, -(-shape[1] // patch) + 1), dtype=np.uint8)
    oy, ox = rng.integers(0, patch, 2)
    return np.repeat(np.repeat(coarse, patch, 0), patch, 1)[oy:oy + shape[0], ox:ox + shape[1]]


def assemble(path, pool, choice, tiled, block):
    """Write a classic little-endian GeoTIFF whose segment k is pool[choice[k]] (LZW, no predictor)."""
    enc = [lzw_encode(p.tobytes()) for p in pool]
    offs, counts = np.empty(len(choice), np.int64), np.empty(len(choice), np.int64)
    with open(path, "wb") as fh:
        fh.write(b"II*\0" + b"\0" * 4)
        pos = 8
        for k, c in enumerate(choice):
            fh.write(enc[c])
            offs[k], counts[k] = pos, len(enc[c])
            pos += len(enc[c])
        pos += pos & 1
        fh.seek(4)
        fh.write(struct.pack("<I", pos))  # the IFD follows the segments
        fh.seek(pos)
        bh, bw = block
        seg_tags = [(322, 3, [bw]), (323, 3, [bh]), (324, 4, offs), (325, 4, counts)] if tiled else [
            (273, 4, offs), (278, 4, [bh]), (279, 4, counts)]
        tags = sorted([(256, 4, [N]), (257, 4, [N]), (258, 3, [8]), (259, 3, [5]), (262, 3, [1]), (277, 3, [1]),
                       (33550, 12, [RES, RES, 0.0]), (33922, 12, [0.0, 0.0, 0.0, X0, Y0 + N * RES, 0.0]),
                       (34735, 3, [1, 1, 0, 2, 1024, 0, 1, 1, 3072, 0, 1, 3035])] + seg_tags)
        data_at = pos + 2 + 12 * len(tags) + 4
        entries, blobs = b"", b""
        for tag, typ, vals in tags:
            body = struct.pack("<" + {3: "H", 4: "I", 12: "d"}[typ] * len(vals), *[v for v in vals])
            e = struct.pack("<HHI", tag, typ, len(vals))
            if len(body) <= 4:
                e += body.ljust(4, b"\0")
            else:
                e += struct.pack("<I", data_at + len(blobs))
                blobs += body
            entries += e
        fh.write(struct.pack("<H", len(tags)) + entries + b"\0" * 4 + blobs)
    return sum(len(enc[c]) for c in choice)


def expected(pool, choice, tiled, block):
    out = np.empty((N, N), np.uint8)
    bh, bw = block
    across = -(-N // bw)
    for k, c in enumerate(choice):
        r0, c0 = (k // across) * bh, (k % across) * bw
        h, w = min(bh, N - r0), min(bw, N - c0)
        out[r0:r0 + h, c0:c0 + w] = pool[c][:h, :w]
    return out


def kernel_ms(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ms = {}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", 0) or 0
        if t and ("tiff" in ev.key or "Memcpy" in ev.key):
            ms[ev.key[:60]] = round(t / 1e3, 2)
    return ms


def best(fn, repeat):
    walls = []
    for _ in range(repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    return round(min(walls) * 1e3, 1), [round(w * 1e3, 1) for w in walls]


def layout(tmp, name, tiled, block, pool_n, repeat, rng):
    pool = [class_map(rng, block) for _ in range(pool_n)]
    bh, bw = block
    n_seg = -(-N // bh) * -(-N // bw)
    choice = rng.integers(0, pool_n, n_seg)
    path = os.path.join(tmp, name + ".tif")
    t0 = time.perf_counter()
    comp_bytes = assemble(path, pool, choice, tiled, block)
    build_s = time.perf_counter() - t0
    want = expected(pool, choice, tiled, block)
    res = dict(segments=int(n_seg), compressed_bytes=int(comp_bytes), ratio=round(N * N / comp_bytes, 1),
               build_s=round(build_s, 1))
    with open(path, "rb") as fh:  # page cache warm-up, then the timed read
        while fh.read(1 << 26):
            pass
    t0 = time.perf_counter()
    with open(path, "rb") as fh:
        blob = fh.read()
    res["file_read_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    pinned = torch.from_numpy(np.frombuffer(blob, np.uint8)).pin_memory()
    dev = torch.empty(len(blob), dtype=torch.uint8, device="cuda")
    res["h2d_compressed_ms"] = best(lambda: dev.copy_(pinned, non_blocking=True), repeat)[0]
    del dev, pinned, blob
    r = geotiff.read(path)  # warm-up, and the check
    want_d = torch.from_numpy(want).to("cuda")
    assert torch.equal(r.array, want_d), f"{name}: decode differs from the assembled raster"
    del r, want_d
    res["read_ms_best"], res["read_ms"] = best(lambda: geotiff.read(path), repeat)
    res["device_ms"] = kernel_ms(lambda: geotiff.read(path))
    res["pageable_upload_of_decoded_ms_best"], res["pageable_upload_of_decoded_ms"] = best(
        lambda: torch.from_numpy(want).to("cuda"), repeat)
    torch.cuda.empty_cache()
    return res, path, want


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pool", type=int, default=48)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--regions", type=int, default=300)
    ap.add_argument("--no-availability", action="store_true")
    ap.add_argument("--out", help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(0)
    out = dict(gpu=gpu, pixels=N * N)
    with tempfile.TemporaryDirectory() as tmp:
        out["striped_1_row"], _, _ = layout(tmp, "striped", False, (1, N), max(4, a.pool // 4), a.repeat, rng)
        out["tiled_256"], path, want = layout(tmp, "tiled", True, (256, 256), a.pool, a.repeat, rng)
        if not a.no_availability:
            import prof_availability as PA

            cut, regions, ex = PA.case(a.regions, 4000)
            arr = gis.Raster(want, (RES, 0.0, X0, 0.0, -RES, Y0 + N * RES), 3035)
            av = {}
            results = {}
            for label, land in (("array", arr), ("geotiff_path", path)):
                walls = []
                for _ in range(a.repeat):
                    ex.rasters[0]["raster"] = land  # each call opens the path afresh
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    A = cut.availabilitymatrix(regions, ex, shapes_crs=3035)
                    torch.cuda.synchronize()
                    walls.append(time.perf_counter() - t0)
                results[label] = np.asarray(A.values)
                av[label] = dict(wall_s_best=round(min(walls), 3), wall_s=[round(w, 3) for w in walls])
            assert np.array_equal(results["array"], results["geotiff_path"]), "path and array availability differ"
            out["availabilitymatrix"] = av
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
