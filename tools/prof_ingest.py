"""Time the GPU inflate against the host decoder on compressed cutouts and Deflate GeoTIFFs.

Cases (each optional, ``--cases a,b,c,d``):
  (a) a Europe-sized cutout: --nx x --ny x --steps, --vars float32 variables, chunk (100, ny, nx),
      zlib 9 + shuffle (the reference's encoding), the file in the page cache.
  (b) the same with chunks of (100, ny/2, nx/2): four times as many, shorter streams.
  (c) the north-star grid 1440 x 720, --c-steps steps, chunk (100, 720, 1440): few, very long streams.
  (d) a --tiff-n x --tiff-n uint8 land-cover raster (prof_geotiff's class maps) as a Deflate GeoTIFF,
      tiled 256 x 256 and in 1-row strips; with --parent, also read by that tree's build (a checkout
      of an earlier version) in a subprocess, alternating with this build.

For (a)-(c) the two routes are, alternating, --repeat times each after a warm-up:
  host:   Cutout(data=lazy.isel_time(0, nt)).to_device()  (host threads decode, pageable upload)
  device: Cutout(lazy).to_device()                          (compressed upload, k_inflate)
Reported: median wall times, file bytes, PCIe bytes, streams, k_inflate time from torch.profiler
(a run of its own), decoded GB/s, and the compression ratio of the synthetic fields.  Files go to a
temporary directory; the card's name and power limit are read in the same run.

    python tools/prof_ingest.py [--cases a,b,c,d] [--steps 8760] [--repeat 3] [--out PATH]
"""

import argparse
import json
import os
import statistics
import struct
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import atlite_b200 as ab  # noqa: E402
from atlite_b200 import geotiff, ingest, synthetic as syn  # noqa: E402


def write_container(path, names, shape, chunk, level=9, pool=8, seed=0):
    """The chunk container of ingest.write_chunked with every chunk drawn from ``pool`` distinct
    compressed chunks (smooth synthetic float32 weather-like fields with small noise, shuffled):
    zlib 9 runs at a few MB/s per core, so a cutout of realistic size is assembled rather than
    compressed chunk by chunk; the decode work per chunk is that of a real one."""
    nt, ny, nx = shape
    ct, cy, cx = chunk
    index = {"format": "atlite_b200-chunks-1", "variables": {}, "attrs": {}, "static": {},
             "coords": {"time": syn.make_time(nt).as_unit("ns").asi8.tolist(),
                        "x": (np.arange(nx) * 0.25 - 12.0).tolist(), "y": (np.arange(ny) * 0.25 + 33.0).tolist()}}

    def encode(p):
        rng = np.random.default_rng([seed, p])
        tt = np.arange(p * ct, (p + 1) * ct, dtype=np.float32)[:, None, None]
        yy, xx = np.mgrid[0:cy, 0:cx].astype(np.float32)
        base = 250.0 + 10.0 * p + 8.0 * np.sin(xx / 23.0 + tt / 24.0) * np.cos(yy / 17.0)
        blk = (base + rng.normal(0, 0.05, base.shape)).astype(np.float32)
        return zlib.compress(ingest.shuffle_bytes(blk), level)

    with ThreadPoolExecutor(min(pool, os.cpu_count())) as ex:
        comp = list(ex.map(encode, range(pool)))
    decoded = 0
    with open(path, "wb") as fh:
        for v, name in enumerate(names):
            jobs = [(t, y, x) for t in range(0, nt, ct) for y in range(0, ny, cy) for x in range(0, nx, cx)]
            offs, sizes = [], []
            for j in range(len(jobs)):
                c = comp[(j + 3 * v) % pool]
                offs.append(fh.tell())
                sizes.append(len(c))
                fh.write(c)
            index["variables"][name] = dict(shape=[nt, ny, nx], chunk=list(chunk), dtype="<f4", shuffle=True,
                                            deflate=True, offsets=offs, sizes=sizes, origins=[list(j) for j in jobs])
            decoded += nt * ny * nx * 4
    with open(path + ".index.json", "w") as fh:
        json.dump(index, fh)
    return decoded


def kernel_ms(fn, key):
    """(summed kernel ms, launches, ms during which at least one such kernel ran) of the kernels
    whose name contains ``key``, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                if key in e.name and str(e.device_type).endswith("CUDA"))
    busy, end = 0.0, None
    for a, b in iv:
        if end is None or a > end:
            busy += b - a
            end = b
        elif b > end:
            busy += b - end
            end = b
    return sum(b - a for a, b in iv) / 1e3, len(iv), busy / 1e3


def alternate(fns, repeat):
    """{name: [wall seconds]} of the functions run in turn, after one warm-up each."""
    walls = {k: [] for k in fns}
    for r in range(repeat + 1):
        for k, fn in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = fn()
            torch.cuda.synchronize()
            if r:
                walls[k].append(time.perf_counter() - t0)
            del res
            torch.cuda.empty_cache()
    return walls


def cutout_case(tmp, name, shape, chunk, n_vars, repeat, pool=8):
    path = os.path.join(tmp, f"{name}.bin")
    names = [f"v{k}" for k in range(n_vars)]
    t0 = time.perf_counter()
    decoded = write_container(path, names, shape, chunk, pool=pool)
    file_bytes = os.path.getsize(path)
    with open(path, "rb") as fh:  # into the page cache
        while fh.read(1 << 26):
            pass
    lazy = ingest.open_cutout(path)
    nt = shape[0]
    host = lambda: ab.Cutout(data=lazy.isel_time(0, nt)).to_device()  # noqa: E731
    dev = lambda: ab.Cutout(data=lazy).to_device()  # noqa: E731
    a, b = host(), dev()
    for n in names:  # the two routes agree bit for bit
        assert torch.equal(a.data.raw(n).view(torch.int32), b.data.raw(n).view(torch.int32)), n
    del a, b
    torch.cuda.empty_cache()
    walls = alternate({"host": host, "device": dev}, repeat)
    k_ms, launches, busy_ms = kernel_ms(dev, "k_inflate")
    streams = sum(len(v.offsets) for v in (lazy._sources[n].var for n in names))
    med = {k: statistics.median(v) for k, v in walls.items()}
    return dict(case=name, shape=list(shape), chunk=list(chunk), variables=n_vars, streams=streams,
                file_bytes=file_bytes, decoded_bytes=decoded, compression_ratio=round(decoded / file_bytes, 3),
                pcie_bytes={"host": decoded, "device": file_bytes},
                wall_s={k: round(v, 3) for k, v in med.items()}, walls_s={k: [round(w, 3) for w in v]
                                                                         for k, v in walls.items()},
                k_inflate_launches=launches, streams_per_launch=round(streams / max(launches, 1), 1),
                k_inflate_summed_ms=round(k_ms, 1), k_inflate_busy_ms=round(busy_ms, 1),
                k_inflate_decoded_GBps=round(decoded / (busy_ms / 1e3) / 1e9, 2) if busy_ms else None,
                # a launch lasts about as long as its slowest stream: bytes per stream over the mean launch
                per_stream_MBps=round(decoded / streams / (k_ms / max(launches, 1) / 1e3) / 1e6, 1) if k_ms else None,
                device_route_decoded_GBps=round(decoded / med["device"] / 1e9, 2),
                host_route_decoded_GBps=round(decoded / med["host"] / 1e9, 2),
                write_s=round(time.perf_counter() - t0, 1))


def class_map(rng, shape, patch=20):
    coarse = rng.integers(0, 44, (-(-shape[0] // patch) + 1, -(-shape[1] // patch) + 1), dtype=np.uint8)
    oy, ox = rng.integers(0, patch, 2)
    return np.repeat(np.repeat(coarse, patch, 0), patch, 1)[oy:oy + shape[0], ox:ox + shape[1]]


def write_deflate_tiff(path, n, tiled, block, pool_n, rng):
    """A classic little-endian uint8 GeoTIFF (EPSG:3035, 100 m) of Deflate segments, each drawn from
    a pool of class-map segments; returns (file bytes, segments)."""
    pool = [zlib.compress(class_map(rng, block).tobytes(), 6) for _ in range(pool_n)]
    bh, bw = block
    n_seg = -(-n // bh) * -(-n // bw)
    choice = rng.integers(0, pool_n, n_seg)
    offs, counts = np.empty(n_seg, np.int64), np.empty(n_seg, np.int64)
    with open(path, "wb") as fh:
        fh.write(b"II*\0" + b"\0" * 4)
        pos = 8
        for k, c in enumerate(choice):
            fh.write(pool[c])
            offs[k], counts[k] = pos, len(pool[c])
            pos += len(pool[c])
        pos += pos & 1
        fh.seek(4)
        fh.write(struct.pack("<I", pos))
        fh.seek(pos)
        seg = [(322, 3, [bw]), (323, 3, [bh]), (324, 4, offs), (325, 4, counts)] if tiled else [
            (273, 4, offs), (278, 4, [bh]), (279, 4, counts)]
        tags = sorted([(256, 4, [n]), (257, 4, [n]), (258, 3, [8]), (259, 3, [8]), (262, 3, [1]), (277, 3, [1]),
                       (33550, 12, [100.0, 100.0, 0.0]), (33922, 12, [0.0, 0.0, 0.0, 2.0e6, 1.0e6 + n * 100.0, 0.0]),
                       (34735, 3, [1, 1, 0, 2, 1024, 0, 1, 1, 3072, 0, 1, 3035])] + seg)
        data_at = pos + 2 + 12 * len(tags) + 4
        entries, blobs = b"", b""
        for tag, typ, vals in tags:
            body = struct.pack("<" + {3: "H", 4: "I", 12: "d"}[typ] * len(vals), *vals)
            e = struct.pack("<HHI", tag, typ, len(vals))
            if len(body) <= 4:
                e += body.ljust(4, b"\0")
            else:
                e += struct.pack("<I", data_at + len(blobs))
                blobs += body
            entries += e
        fh.write(struct.pack("<H", len(tags)) + entries + b"\0" * 4 + blobs)
    return os.path.getsize(path), n_seg


PARENT_READ = """
import sys, time, torch
sys.path.insert(0, sys.argv[1])
from atlite_b200 import geotiff
walls = []
for r in range(int(sys.argv[3]) + 1):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    a = geotiff.read(sys.argv[2]); torch.cuda.synchronize()
    if r: walls.append(time.perf_counter() - t0)
    del a
print(",".join(str(w) for w in walls))
"""


def tiff_case(tmp, n, tiled, repeat, parent, rng):
    block = (256, 256) if tiled else (1, n)
    path = os.path.join(tmp, f"lc_deflate_{'tiled' if tiled else 'strips'}.tif")
    file_bytes, n_seg = write_deflate_tiff(path, n, tiled, block, 48, rng)
    with open(path, "rb") as fh:
        while fh.read(1 << 26):
            pass
    this = lambda: geotiff.read(path)  # noqa: E731
    walls = alternate({"this": this}, 0)  # warm-up only
    walls = {"this": [], "parent": []}
    for _ in range(repeat):
        walls["this"] += alternate({"this": this}, 1)["this"]
        if parent:
            r = subprocess.run([sys.executable, "-c", PARENT_READ, parent, path, "1"], capture_output=True, text=True)
            if r.returncode:
                raise RuntimeError(r.stderr[-2000:])
            walls["parent"] += [float(v) for v in r.stdout.strip().split(",")]
    k_ms, launches, busy_ms = kernel_ms(this, "k_inflate")
    decoded = n * n
    med = {k: statistics.median(v) for k, v in walls.items() if v}
    return dict(case="d", layout="tiled 256x256" if tiled else "1-row strips", pixels=decoded, streams=n_seg,
                file_bytes=file_bytes, compression_ratio=round(decoded / file_bytes, 2),
                pcie_bytes={"this": file_bytes, "parent": decoded},
                wall_s={k: round(v, 3) for k, v in med.items()}, walls_s={k: [round(w, 3) for w in v]
                                                                         for k, v in walls.items()},
                k_inflate_launches=launches, k_inflate_busy_ms=round(busy_ms, 1),
                k_inflate_decoded_GBps=round(decoded / (busy_ms / 1e3) / 1e9, 2) if busy_ms else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="a,b,c,d")
    ap.add_argument("--nx", type=int, default=281)
    ap.add_argument("--ny", type=int, default=201)
    ap.add_argument("--steps", type=int, default=8760)
    ap.add_argument("--vars", type=int, default=10)
    ap.add_argument("--c-steps", type=int, default=0, help="steps of case c (0: what fits 80%% of device memory)")
    ap.add_argument("--tiff-n", type=int, default=40000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built tree of an earlier version, for case d")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = dict(gpu=gpu, cpus=os.cpu_count(), results=[])
    cases = a.cases.split(",")
    with tempfile.TemporaryDirectory() as tmp:
        if "a" in cases:
            res["results"].append(cutout_case(tmp, "a", (a.steps, a.ny, a.nx), (100, a.ny, a.nx), a.vars, a.repeat))
            print(json.dumps(res["results"][-1]), flush=True)
        if "b" in cases:
            ch = (100, -(-a.ny // 2), -(-a.nx // 2))
            res["results"].append(cutout_case(tmp, "b", (a.steps, a.ny, a.nx), ch, a.vars, a.repeat))
            print(json.dumps(res["results"][-1]), flush=True)
        for f in os.listdir(tmp):
            os.remove(os.path.join(tmp, f))
        if "c" in cases:
            free = torch.cuda.mem_get_info()[1] * 0.8
            steps = a.c_steps or int(free // (1440 * 720 * 4) // 100 * 100)  # one variable, decoded
            res["results"].append(cutout_case(tmp, "c", (steps, 720, 1440), (100, 720, 1440), 1, a.repeat, pool=2))
            print(json.dumps(res["results"][-1]), flush=True)
        for f in os.listdir(tmp):
            os.remove(os.path.join(tmp, f))
        if "d" in cases:
            rng = np.random.default_rng(0)
            for tiled in (True, False):
                res["results"].append(tiff_case(tmp, a.tiff_n, tiled, a.repeat, a.parent, rng))
                print(json.dumps(res["results"][-1]), flush=True)
    print(json.dumps(dict(gpu=gpu, cpus=res["cpus"])))
    if a.out:
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
