"""Write the GeoTIFF fixtures of tests/test_geotiff.py with libtiff, and the arrays libtiff decodes.

Pillow (built against libtiff) writes striped files with ``compression=`` and a ``tiffinfo`` that
carries the predictor (317), rows per strip (278), ModelPixelScale (33550), ModelTiepoint (33922),
the GeoKeyDirectory (34735) and GDAL_NODATA (42113); OpenCV's bundled libtiff reads every file back
into ``reference_geotiff.npz`` (key: the file's stem).  Tiled, BigTIFF and big-endian files come
from the test file's own writer instead, since Pillow writes none of them.

    python tests/golden/make_golden_geotiff.py
"""

import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "geotiff")


def geokeys(epsg, geographic=False, point=False):
    """GeoKeyDirectory: model type, raster type, then the projected or geographic CRS key."""
    keys = [(1024, 2 if geographic else 1), (1025, 2 if point else 1), (2048 if geographic else 3072, epsg)]
    d = [1, 1, 0, len(keys)]
    for k, v in keys:
        d += [k, 0, 1, v]
    return tuple(d)


def blocky(rng, shape, classes, patch):
    coarse = rng.integers(0, classes, (-(-shape[0] // patch), -(-shape[1] // patch)))
    return np.repeat(np.repeat(coarse, patch, 0), patch, 1)[:shape[0], :shape[1]]


def cases():
    rng = np.random.default_rng(7)
    lc = blocky(rng, (97, 131), 44, 6).astype(np.uint8)
    lc[rng.random(lc.shape) < 0.02] = 255
    depth = (blocky(rng, (61, 83), 50, 5) * -7.5 + rng.normal(0, 2, (61, 83))).astype(np.float32)
    u16 = (blocky(rng, (45, 70), 3000, 3) + rng.integers(0, 40, (45, 70))).astype(np.uint16)
    i32 = (rng.integers(-100000, 100000, (33, 41))).astype(np.int32)
    noise = rng.integers(0, 256, (150, 211)).astype(np.uint8)  # many Clears at the 12-bit limit
    utm = (3072, 100.0, 500000.0, 5600000.0)
    return [
        # name, array, compression, predictor, rows per strip, (epsg, geographic, point), scale, origin, nodata
        ("lc_u8_lzw_p2_3035", lc, "tiff_lzw", 2, 7, (3035, False, False), 100.0, (4.0e6, 3.1e6), "255"),
        ("lc_u8_lzw_p1_3035", lc, "tiff_lzw", 1, 16, (3035, False, False), 100.0, (4.0e6, 3.1e6), None),
        ("lc_u8_deflate_p2_3035", lc, "tiff_adobe_deflate", 2, 10, (3035, False, False), 100.0, (4.0e6, 3.1e6), None),
        ("lc_u8_none_4326_point", lc, "raw", 1, 13, (4326, True, True), 0.01, (5.0, 47.0), "0"),
        ("noise_u8_lzw_p1_4326", noise, "tiff_lzw", 1, 150, (4326, True, False), 0.01, (5.0, 47.0), None),
        ("u16_lzw_p2_3035", u16, "tiff_lzw", 2, 4, (3035, False, False), 250.0, (3.9e6, 3.0e6), "65535"),
        ("u16_deflate_p1_3035", u16, "tiff_adobe_deflate", 1, 45, (3035, False, False), 250.0, (3.9e6, 3.0e6), None),
        ("i32_none_p1_4326", i32, "raw", 1, 9, (4326, True, False), 0.25, (-10.0, 60.0), "-9999"),
        ("i32_lzw_p2_4326", i32, "tiff_lzw", 2, 1, (4326, True, False), 0.25, (-10.0, 60.0), None),
        ("depth_f32_lzw_p3_4326", depth, "tiff_lzw", 3, 8, (4326, True, False), 0.01, (5.0, 47.0), "nan"),
        ("depth_f32_deflate_p3_4326", depth, "tiff_adobe_deflate", 3, 61, (4326, True, False), 0.01, (5.0, 47.0),
         None),
        ("depth_f32_lzw_p2_4326", depth, "tiff_lzw", 2, 5, (4326, True, False), 0.01, (5.0, 47.0), "-3.5e38"),
        ("lc_u8_lzw_p2_userdefined", lc, "tiff_lzw", 2, 32, (32767, False, False), utm[1], utm[2:], None),
    ]


def main():
    import cv2
    from PIL import Image, TiffImagePlugin

    os.makedirs(OUT, exist_ok=True)
    arrays = {}
    for name, arr, comp, pred, rps, (epsg, geo, point), scale, (x0, y0), nodata in cases():
        ifd = TiffImagePlugin.ImageFileDirectory_v2()
        ifd[317] = pred
        ifd[278] = rps
        ifd[33550], ifd.tagtype[33550] = (scale, scale, 0.0), 12
        ifd[33922], ifd.tagtype[33922] = (0.0, 0.0, 0.0, x0, y0, 0.0), 12
        ifd[34735], ifd.tagtype[34735] = geokeys(epsg, geo, point), 3
        if nodata is not None:
            ifd[42113], ifd.tagtype[42113] = nodata, 2
        path = os.path.join(OUT, name + ".tif")
        Image.fromarray(arr).save(path, compression=comp, tiffinfo=ifd)
        back = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        assert back is not None and back.dtype == arr.dtype and np.array_equal(back, arr, equal_nan=True), name
        arrays[name] = back
    np.savez_compressed(os.path.join(HERE, "reference_geotiff.npz"), **arrays)
    print(f"wrote {len(arrays)} GeoTIFFs under {OUT}")


if __name__ == "__main__":
    main()
