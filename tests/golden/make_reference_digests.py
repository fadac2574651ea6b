"""Writes tests/golden/reference_digests.json and tests/golden/images/: what the reference produced for every case the
tests compare against it, so that those comparisons also run where the reference is not built.

  reference_digests.json   SHA-256 digests (tests/util.py: array_digest / bytes_digest) of the reference's results on
                           the tests' own seeded inputs:
                             convert/<src>/<dst>           tools/halide_image_io.h element conversion (test_image_io)
                             save/<fmt>/<type>/<shape>     the file save_image writes (FORMAT_CASES and TIFF_CASES)
                             autosave/<fmt>/<type>/<shape> the image the reference reads back from convert_and_save_image's file
                             loadconv/<image>/<type>       load_and_convert_image of the images below
                             ref_blur/<h>x<w>/<fast>       apps/blur/test.cpp's C blur (naive 0, SSE 1)
                             png_crop/<image>              the crop below of the reference's PNG as decoded in full
  images/                  matrix_3200.mat, matrix_7000.mat and gray_small.png as apps/images ships them;
                           gray_crop.pgm, a 128x96 crop of gray_small.pgm written by the reference's own pgm writer;
                           rgb_crop.png, a 128x96 crop of rgb_small.png (an 8-bit RGB PNG written by halide_b200.image_io);
                           PNG_CROPS: 96x64 crops of rgb_small.png, rgb_small16.png and bayer_small.png written by OpenCV
                           (8-bit RGB, 16-bit RGB, 16-bit gray), an encoder independent of halide_b200.image_io

Run from the repository root after build() has built oracle/_ref (it needs the reference source tree):
  python tests/golden/make_reference_digests.py <reference source tree>"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_image_io import (AUTOSAVE_SHAPES, FORMAT_CASES, IMAGES, LOADCONV_CASES, NAMES, PNG_CROPS, REF, TIFF_CASES,  # noqa: E402
                           format_case_key, random_image, read_dump, ref_convert, samples, write_dump)
from util import array_digest, bytes_digest, u16_frame  # noqa: E402

from oracle import pyoracle  # noqa: E402


def make_images(ref_images, d, out):
    import cv2
    os.makedirs(IMAGES, exist_ok=True)
    for name in ("matrix_3200.mat", "matrix_7000.mat", "gray_small.png"):
        shutil.copyfile(os.path.join(ref_images, name), os.path.join(IMAGES, name))
    subprocess.run([REF, "load", os.path.join(ref_images, "gray_small.pgm"), os.path.join(d, "g.dump")], check=True)
    write_dump(np.ascontiguousarray(read_dump(os.path.join(d, "g.dump"))[:96, :128]), os.path.join(d, "crop.dump"))
    subprocess.run([REF, "save", os.path.join(d, "crop.dump"), os.path.join(IMAGES, "gray_crop.pgm")], check=True)
    from halide_b200 import image_io
    image_io.save(np.ascontiguousarray(image_io.load(os.path.join(ref_images, "rgb_small.png"))[:, :96, :128]),
                  os.path.join(IMAGES, "rgb_crop.png"))
    for crop, src in PNG_CROPS.items():
        full = os.path.join(ref_images, src)
        os.environ["HALIDE_B200_PNG_PURE"] = "1"
        try:
            pure = image_io.load(full)
        finally:
            del os.environ["HALIDE_B200_PNG_PURE"]
        assert np.array_equal(pure, image_io.load(full)), src
        a = np.ascontiguousarray(pure[..., :64, :96])
        cv2.imwrite(os.path.join(IMAGES, crop), a if a.ndim == 2 else np.ascontiguousarray(a.transpose(1, 2, 0)[:, :, ::-1]))
        out[f"png_crop/{crop}"] = array_digest(a)


def main(ref_tree):
    from pathlib import Path
    out = {}
    with tempfile.TemporaryDirectory() as d:
        make_images(os.path.join(ref_tree, "apps", "images"), d, out)
        tmp = Path(d)
        for src in NAMES:   # test_convert_matches_reference_for_every_target
            a = samples(NAMES[src], seed=len(src))
            for dst in NAMES:
                out[f"convert/{src}/{dst}"] = array_digest(ref_convert(a, dst, tmp))
        for fmt, dtype, shape in FORMAT_CASES:   # test_formats_round_trip_through_the_reference
            a = random_image(dtype, shape, len(shape) * 7 + np.dtype(dtype).itemsize)
            write_dump(a, os.path.join(d, "a.dump"))
            path = os.path.join(d, "img." + fmt)
            subprocess.run([REF, "save", os.path.join(d, "a.dump"), path], check=True)
            out["save/" + format_case_key(fmt, dtype, shape)] = bytes_digest(open(path, "rb").read())
        for dtype, shape in TIFF_CASES:   # test_tiff_writer_is_byte_identical
            write_dump(random_image(dtype, shape, 11), os.path.join(d, "a.dump"))
            subprocess.run([REF, "save", os.path.join(d, "a.dump"), os.path.join(d, "ref.tiff")], check=True)
            out["save/" + format_case_key("tiff", dtype, shape)] = bytes_digest(open(os.path.join(d, "ref.tiff"), "rb").read())
        for fmt, shapes in AUTOSAVE_SHAPES.items():   # test_convert_and_save_picks_the_reference_type
            for shape in shapes:
                for src in NAMES.values():
                    write_dump(random_image(src, shape, 3), os.path.join(d, "a.dump"))
                    subprocess.run([REF, "autosave", os.path.join(d, "a.dump"), os.path.join(d, "ref." + fmt)], check=True)
                    subprocess.run([REF, "load", os.path.join(d, "ref." + fmt), os.path.join(d, "r.dump")], check=True)
                    out["autosave/" + format_case_key(fmt, src, shape)] = array_digest(read_dump(os.path.join(d, "r.dump")))
        for name, types in LOADCONV_CASES:   # test_load_and_convert_of_the_reference_images
            for t in types:
                subprocess.run([REF, "loadconv", os.path.join(IMAGES, name), t, os.path.join(d, "x.dump")], check=True)
                out[f"loadconv/{name}/{t}"] = array_digest(read_dump(os.path.join(d, "x.dump")))
        # test_reference_png_images_decode_the_same_both_ways: gray_small.png must decode to gray_small.pgm
        subprocess.run([REF, "loadconv", os.path.join(ref_tree, "apps", "images", "gray_small.pgm"), "u8", os.path.join(d, "x.dump")],
                       check=True)
        out["loadconv/gray_small.pgm/u8"] = array_digest(read_dump(os.path.join(d, "x.dump")))
    # test_blur_oracle_matches_reference_c_implementation and test_blur_matches_reference_c_on_harness_shape
    rng = np.random.default_rng(11)
    small = (rng.integers(0, 65536, (98, 264), dtype=np.uint16) & 0xFFF).astype(np.uint16)
    harness = u16_frame((1922, 2568), 7, bits=12)
    for fast in (0, 1):
        out[f"ref_blur/98x264/{fast}"] = array_digest(pyoracle.ref_blur(small, bool(fast)))
        out[f"ref_blur/1922x2568/{fast}"] = array_digest(pyoracle.ref_blur(harness, bool(fast)))
    with open(os.path.join(ROOT, "tests", "golden", "reference_digests.json"), "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "digests")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
