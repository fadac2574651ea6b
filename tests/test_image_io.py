"""halide_b200/image_io.py against the reference's own image I/O header (tools/halide_image_io.h), which is compiled in
place into oracle/_ref/ref_image_io (oracle/ref_image_io_tool.cpp): element conversions for every type pair, every
format both ways (the reference writes / we read, we write / the reference reads), and the type / dimensionality choice
of convert_and_save_image.  Where the reference binary is not available (oracle/_ref is built only where the reference
source tree is), what it produced for every one of these cases stands in for it: SHA-256 digests in
tests/golden/reference_digests.json (tests/golden/make_reference_digests.py) and the golden vectors of
tests/golden/image_io_golden.npz (tests/golden/make_image_io_golden.py), both made with the same binary."""
import os
import subprocess

import numpy as np
import pytest
from util import array_digest, bytes_digest, reference_digest

from halide_b200 import image_io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "ref_image_io")
GOLDEN = os.path.join(ROOT, "tests", "golden", "image_io_golden.npz")
NAMES = {"u8": np.uint8, "u16": np.uint16, "u32": np.uint32, "u64": np.uint64, "i8": np.int8, "i16": np.int16,
         "i32": np.int32, "i64": np.int64, "f32": np.float32, "f64": np.float64}
TNAME = {np.dtype(v): k for k, v in NAMES.items()}
IMAGES = os.path.join(ROOT, "tests", "golden", "images")   # small images from the reference's apps/images
HAVE_REF = os.path.exists(REF)


def samples(dtype, n=2048, seed=0):
    """Inputs with defined behaviour in the reference: every integer pattern; floats mostly in [0, 1] plus exact halves,
    negatives and values up to a few thousand (float -> integer conversions go through lround and a modular cast)."""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt.kind in "ui":
        info = np.iinfo(dt)
        edge = np.array([info.min, info.max, 0, 1, info.max // 2, info.max // 2 + 1, info.min // 2, 127, 128, 255, 256 % (info.max + 1)],
                        dtype=np.int64 if dt.kind == "i" else np.uint64).astype(dt)
        body = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        return np.concatenate([edge, body])
    edge = np.array([0.0, 1.0, 0.5, 0.25, 0.75, 1.0 / 255, 0.5 / 255, 1.5 / 255, 2.5 / 255, 0.5 / 65535, 1.5 / 65535, -0.25, -1.0, 1.5,
                     2.0, 100.25, 1000.5, -3.75], dtype=dt)
    return np.concatenate([edge, rng.random(n).astype(dt), (rng.random(64) * 8 - 4).astype(dt)])


def ref_convert(a, dst, tmp_path):
    src_f, dst_f = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    a.tofile(src_f)
    subprocess.run([REF, "convert", TNAME[a.dtype], dst, src_f, dst_f], check=True)
    return np.fromfile(dst_f, dtype=NAMES[dst])


def write_dump(a, path):
    with open(path, "wb") as f:
        f.write((" ".join([TNAME[a.dtype], str(a.ndim)] + [str(e) for e in reversed(a.shape)]) + "\n").encode())
        f.write(np.ascontiguousarray(a).tobytes())


def read_dump(path):
    b = open(path, "rb").read()
    nl = b.index(b"\n")
    parts = b[:nl].decode().split()
    ext = [int(e) for e in parts[2:2 + int(parts[1])]]
    return np.frombuffer(b[nl + 1:], dtype=NAMES[parts[0]]).reshape(tuple(reversed(ext))).copy()


@pytest.mark.parametrize("src", list(NAMES))
def test_convert_matches_reference_for_every_target(src, tmp_path):
    a = samples(NAMES[src], seed=len(src))
    for dst in NAMES:
        got = image_io.convert(a, NAMES[dst])
        if not HAVE_REF:
            assert array_digest(got) == reference_digest(f"convert/{src}/{dst}"), (src, dst)
            continue
        want = ref_convert(a, dst, tmp_path)
        assert got.dtype == want.dtype
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (src, dst, a[np.flatnonzero(got != want)[:4]])


def test_convert_matches_golden_vectors():
    g = np.load(GOLDEN)
    for key in g.files:
        if not key.startswith("conv_in_"):
            continue
        src = key[len("conv_in_"):]
        for dst in NAMES:
            want = g[f"conv_{src}_{dst}"]
            got = image_io.convert(g[key], NAMES[dst])
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (src, dst)


def test_conversion_rules_spelled_out():
    """The rules the natural-image runs of the seven pipelines actually meet (tools/halide_image_io.h:130-240,606-616)."""
    u8 = np.arange(256, dtype=np.uint8)
    assert np.array_equal(image_io.convert(u8, np.uint16), u8.astype(np.uint16) * 257)
    assert np.array_equal(image_io.convert(image_io.convert(u8, np.uint16), np.uint8), u8)
    u16 = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    assert np.array_equal(image_io.convert(u16, np.uint8), np.floor((u16.astype(np.float64) + 128.5) / 257).astype(np.uint8))
    assert image_io.convert(u8, np.float32)[255] == np.float32(1.0) and image_io.convert(u16, np.float32)[65535] == np.float32(1.0)
    f = np.array([0.0, 0.5 / 255, 1.5 / 255 + 1e-7, 1.0, 2.0, -1.0 / 255], np.float32)
    assert list(image_io.convert(f, np.uint8)) == [0, 1, 2, 255, 254, 255]   # lround, then a modular cast


FORMAT_CASES = [("pgm", np.uint8, (37, 50)), ("pgm", np.uint16, (9, 13)), ("ppm", np.uint8, (3, 21, 34)), ("ppm", np.uint16, (3, 5, 7)),
                ("npy", np.float32, (3, 6, 5)), ("npy", np.uint16, (4, 9)), ("npy", np.int64, (2, 3, 4, 5)), ("npy", np.uint8, (11,)),
                ("tmp", np.float32, (1, 3, 8, 6)), ("tmp", np.int16, (2, 2, 3, 4)), ("mat", np.float32, (3, 4)),
                ("mat", np.float64, (2, 3, 5)), ("mat", np.uint16, (4, 6))]


def random_image(dtype, shape, seed):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt.kind == "f":
        return rng.random(shape).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, shape, dtype=dt, endpoint=True)


def format_case_key(fmt, dtype, shape):
    return f"{fmt}/{TNAME[np.dtype(dtype)]}/{'x'.join(map(str, shape))}"


@pytest.mark.parametrize("fmt,dtype,shape", FORMAT_CASES)
def test_formats_round_trip_through_the_reference(fmt, dtype, shape, tmp_path):
    a = random_image(dtype, shape, len(shape) * 7 + np.dtype(dtype).itemsize)
    (tmp_path / "r").mkdir()
    (tmp_path / "o").mkdir()
    # (same base name in two directories: a .mat file carries its own file name as the variable name)
    dump, ref_file, our_file, back = (str(tmp_path / n) for n in ("a.dump", "r/img." + fmt, "o/img." + fmt, "b.dump"))
    if not HAVE_REF:
        # every format here is written byte for byte as the reference writes it, so our file stands for the reference's
        image_io.save(a, our_file)
        assert bytes_digest(open(our_file, "rb").read()) == reference_digest("save/" + format_case_key(fmt, dtype, shape))
        got = image_io.load(our_file)
        assert got.dtype == a.dtype and np.array_equal(got, a)
        return
    # the reference writes, we read
    write_dump(a, dump)
    subprocess.run([REF, "save", dump, ref_file], check=True)
    got = image_io.load(ref_file)
    assert got.dtype == a.dtype and np.array_equal(got, a)
    # we write, the reference reads
    image_io.save(a, our_file)
    subprocess.run([REF, "load", our_file, back], check=True)
    assert np.array_equal(read_dump(back), a)
    if fmt in ("pgm", "ppm", "npy", "tmp", "mat"):   # these writers are byte-for-byte the reference's
        assert open(our_file, "rb").read() == open(ref_file, "rb").read()


AUTOSAVE_SHAPES = {"pgm": [(6, 7)], "ppm": [(3, 6, 7)], "npy": [(5,), (6, 7), (3, 6, 7)], "tmp": [(6, 7), (3, 6, 7), (2, 3, 6, 7)],
                   "mat": [(6, 7), (3, 6, 7)]}


@pytest.mark.parametrize("fmt", ["pgm", "ppm", "npy", "tmp", "mat"])
def test_convert_and_save_picks_the_reference_type(fmt, tmp_path):
    for shape in AUTOSAVE_SHAPES[fmt]:
        for src in NAMES.values():
            a = random_image(src, shape, 3)
            dump, ref_file, our_file, d1, d2 = (str(tmp_path / n) for n in ("a.dump", "ref." + fmt, "ours." + fmt, "r.dump", "o.dump"))
            if not HAVE_REF:
                # what the reference's reader found in the file its convert_and_save_image wrote, against ours read back
                image_io.convert_and_save_image(a, our_file)
                assert array_digest(image_io.load(our_file)) == reference_digest("autosave/" + format_case_key(fmt, src, shape)), \
                    (fmt, shape, src)
                continue
            write_dump(a, dump)
            subprocess.run([REF, "autosave", dump, ref_file], check=True)
            image_io.convert_and_save_image(a, our_file)
            subprocess.run([REF, "load", ref_file, d1], check=True)
            subprocess.run([REF, "load", our_file, d2], check=True)
            want, got = read_dump(d1), read_dump(d2)
            assert got.dtype == want.dtype and got.shape == want.shape, (fmt, shape, src, got.dtype, want.dtype)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (fmt, shape, src)


LOADCONV_CASES = (("gray_crop.pgm", ("u8", "u16", "f32")), ("matrix_3200.mat", ("f32",)), ("matrix_7000.mat", ("f32", "f64")))


def test_load_and_convert_of_the_reference_images(tmp_path):
    """A crop of apps/images/gray_small.pgm (written by the reference) and the camera_pipe colour matrices, loaded into
    every type the harnesses ask for."""
    for name, types in LOADCONV_CASES:
        for t in types:
            got = image_io.load_and_convert_image(os.path.join(IMAGES, name), NAMES[t])
            if not HAVE_REF:
                assert array_digest(got) == reference_digest(f"loadconv/{name}/{t}"), (name, t)
                continue
            out = str(tmp_path / "x.dump")
            subprocess.run([REF, "loadconv", os.path.join(IMAGES, name), t, out], check=True)
            want = read_dump(out)
            assert got.dtype == want.dtype and np.array_equal(got, want), (name, t)


def test_golden_files_decode_identically():
    """Files written by the reference (committed bytes) decode to the committed arrays, and our writers reproduce the
    reference's bytes for the formats whose encoding is fully determined."""
    g = np.load(GOLDEN)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        for key in g.files:
            if not key.startswith("file_"):
                continue
            _, fmt, tag = key.split("_", 2)
            path = os.path.join(d, f"{tag}.{fmt}")
            open(path, "wb").write(g[key].tobytes())
            want = g[f"array_{fmt}_{tag}"]
            got = image_io.load(path)
            assert got.dtype == want.dtype and np.array_equal(got, want), key
            if fmt in ("pgm", "ppm", "npy", "tmp"):
                ours = os.path.join(d, f"ours_{tag}.{fmt}")
                image_io.save(want, ours)
                assert open(ours, "rb").read() == g[key].tobytes(), key


def test_png_codec_round_trip_and_cross_check(tmp_path):
    """PNG (the reference reads it through libpng, which is not available to its header build here): our writer / reader
    round trip for 8- and 16-bit gray, gray+alpha, RGB and RGBA, the pure-Python decoder against OpenCV's on files with
    Sub / Up / Average / Paeth rows when OpenCV is importable."""
    for dtype, shape in ((np.uint8, (20, 31)), (np.uint16, (7, 9)), (np.uint8, (3, 12, 17)), (np.uint16, (3, 6, 5)),
                         (np.uint8, (4, 5, 6)), (np.uint16, (2, 5, 6))):
        a = random_image(dtype, shape, 5)
        p = str(tmp_path / "a.png")
        image_io.save(a, p) if (np.dtype(dtype), len(shape)) in image_io.save_query(p) and (len(shape) == 2 or shape[0] == 3) \
            else image_io._save_png(a, p)
        os.environ["HALIDE_B200_PNG_PURE"] = "1"
        try:
            got = image_io.load(p)
        finally:
            del os.environ["HALIDE_B200_PNG_PURE"]
        assert got.dtype == a.dtype and np.array_equal(got, a), (dtype, shape)
    try:
        import cv2
    except Exception:
        return
    yy, xx = np.mgrid[0:40, 0:56]
    smooth = ((np.sin(xx / 5.0) * np.cos(yy / 7.0) * 0.4 + 0.5) * 65535).astype(np.uint16)   # adaptive filters pick Paeth / Average here
    for arr in (smooth, (smooth >> 8).astype(np.uint8), np.stack([smooth, smooth[::-1], smooth.T[:40, :40].repeat(2, 1)[:, :56]])):
        p = str(tmp_path / "cv.png")
        cv2.imwrite(p, arr if arr.ndim == 2 else np.ascontiguousarray(arr.transpose(1, 2, 0)[:, :, ::-1]))
        os.environ["HALIDE_B200_PNG_PURE"] = "1"
        try:
            pure = image_io.load(p)
        finally:
            del os.environ["HALIDE_B200_PNG_PURE"]
        assert np.array_equal(pure, arr) and np.array_equal(image_io.load(p), arr)


# crops of the reference's sample images apps/images/*_small*.png, re-encoded by OpenCV (tests/golden/make_reference_digests.py)
PNG_CROPS = {"rgb_small_crop.png": "rgb_small.png", "rgb_small16_crop.png": "rgb_small16.png", "bayer_small_crop.png": "bayer_small.png"}


def test_reference_png_images_decode_the_same_both_ways():
    """The reference's sample images through the pure-Python decoder and through OpenCV: gray_small.png (8-bit gray, as
    the reference ships it) and crops of rgb_small.png, rgb_small16.png and bayer_small.png (8-bit RGB, 16-bit RGB,
    16-bit Bayer raw, encoded by OpenCV).  gray_small.png must equal gray_small.pgm as the reference's own reader decodes
    it, and each crop the same region of the reference's PNG decoded in full."""
    try:
        import cv2  # noqa: F401
    except Exception:
        pytest.skip("OpenCV not importable: nothing to cross-check against")
    for name in ("gray_small.png",) + tuple(PNG_CROPS):
        p = os.path.join(IMAGES, name)
        fast = image_io.load(p)
        os.environ["HALIDE_B200_PNG_PURE"] = "1"
        try:
            pure = image_io.load(p)
        finally:
            del os.environ["HALIDE_B200_PNG_PURE"]
        assert fast.dtype == pure.dtype and np.array_equal(fast, pure), name
        if name in PNG_CROPS:
            assert array_digest(pure) == reference_digest(f"png_crop/{name}"), name
    assert array_digest(image_io.load(os.path.join(IMAGES, "gray_small.png"))) == reference_digest("loadconv/gray_small.pgm/u8")


TIFF_CASES = [(np.uint8, (9, 14)), (np.uint16, (3, 9, 14)), (np.float32, (4, 5, 6)), (np.int32, (7,)), (np.float64, (2, 3, 4, 5)),
              (np.uint8, (6, 3, 4)), (np.int16, (1, 2, 8, 9))]


@pytest.mark.parametrize("dtype,shape", TIFF_CASES)
def test_tiff_writer_is_byte_identical(dtype, shape, tmp_path):
    """The reference writes (uncompressed, planar) TIFF and cannot read it back; ours must produce the same bytes —
    including the rule that folds a third dimension below 5 into the channel count."""
    a = random_image(dtype, shape, 11)
    dump, ref_file, our_file = (str(tmp_path / n) for n in ("a.dump", "ref.tiff", "ours.tiff"))
    image_io.save(a, our_file)
    if HAVE_REF:
        write_dump(a, dump)
        subprocess.run([REF, "save", dump, ref_file], check=True)
        assert open(our_file, "rb").read() == open(ref_file, "rb").read()
    else:
        assert bytes_digest(open(our_file, "rb").read()) == reference_digest("save/" + format_case_key("tiff", dtype, shape))
    with pytest.raises(ValueError):
        image_io.load(our_file)


def test_natural_image_flow_like_process_cpp(tmp_path):
    """apps/local_laplacian/process.cpp end to end on the host side: load_and_convert_image(png) into uint16 planes, the
    filter (the CPU oracle stands in for it here — the GPU parity tests cover the filter itself), convert_and_save_image
    to a 16-bit PNG, reload: the file holds exactly the filter's output, and an 8-bit source enters as x * 257."""
    from oracle import pyoracle
    src = os.path.join(IMAGES, "rgb_crop.png")   # a 128x96 crop of apps/images/rgb_small.png
    native = image_io.load(src)
    assert native.dtype == np.uint8 and native.ndim == 3 and native.shape[0] == 3
    frame = image_io.load_and_convert_image(src, np.uint16)
    assert np.array_equal(frame, native.astype(np.uint16) * 257)
    frame = np.ascontiguousarray(frame[:, :96, :128])   # a crop keeps the oracle quick
    out = pyoracle.local_laplacian(frame, 8, 1.0 / 7.0, 1.0)
    dst = str(tmp_path / "out.png")
    image_io.convert_and_save_image(out, dst)
    back = image_io.load(dst)
    assert back.dtype == np.uint16 and np.array_equal(back, out)
    image_io.convert_and_save_image(out, str(tmp_path / "out8.ppm"))   # (.ppm holds uint16 too: saved as is)
    assert np.array_equal(image_io.load(str(tmp_path / "out8.ppm")), out)
