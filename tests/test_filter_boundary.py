"""The C boundary every filter shares: metadata records, argument checks and bounds queries, through every entry point
(F, F_argv, F_auto_schedule, F_auto_schedule_argv, and halide_b200_local_laplacian_sharded next to local_laplacian).

Every CPU case here returns before the library makes a CUDA call, so none needs a GPU.  The expected return codes,
halide_error messages, proposed shapes and metadata contents are literal tables at the end of this file.  They pin the
checks of a Halide-generated prologue (src/AddImageChecks.cpp) as this library reproduces them, including which fault
each filter reports first when two occur at once.  The GPU case checks that the four entry points of a filter compute
the same bits, which is what shows that the argv unpacking delivers the scalars to the kernels."""
import ctypes

import numpy as np
import pytest

U8, U16, F32 = np.uint8, np.uint16, np.float32
I32, F = ctypes.c_int32, ctypes.c_float

# Arguments in ABI order: a buffer is (name, dtype, numpy shape (outermost first), Halide mins or None), a scalar is
# (name, ctype, value).  The values describe a call that passes every check; the last argument is the output.
FILTERS = {
    "halide_blur": [("input", U16, (12, 18), (2, 3)), ("blur_y", U16, (10, 16), (2, 3))],
    "local_laplacian": [("input", U16, (3, 8, 10), None), ("levels", I32, 8), ("alpha", F, 1 / 7), ("beta", F, 1.0),
                        ("output", U16, (3, 8, 10), None)],
    "bilateral_grid": [("input", F32, (8, 10), (1, 2)), ("r_sigma", F, 0.1), ("bilateral_grid", F32, (8, 10), (1, 2))],
    "nl_means": [("input", F32, (3, 8, 10), None), ("patch_size", I32, 3), ("search_area", I32, 7), ("sigma", F, 0.12),
                 ("non_local_means", F32, (3, 8, 10), None)],
    "stencil_chain": [("input", U16, (8, 10), None), ("output", U16, (8, 10), None)],
    "camera_pipe": [("input", U16, (44, 52), (10, 6)), ("matrix_3200", F32, (3, 4), None), ("matrix_7000", F32, (3, 4), None),
                    ("color_temp", F, 3700.0), ("gamma", F, 2.0), ("contrast", F, 50.0), ("sharpen_strength", F, 1.0),
                    ("blackLevel", I32, 25), ("whiteLevel", I32, 1023), ("processed", U8, (3, 32, 40), None)],
    "conv_layer": [("input", F32, (5, 82, 102, 128), None), ("filter", F32, (128, 3, 3, 128), None), ("bias", F32, (128,), None),
                   ("relu", F32, (5, 80, 100, 128), None)],
}
SHARDED = "halide_b200_local_laplacian_sharded"
FILTERS[SHARDED] = FILTERS["local_laplacian"] + [("frame_y_min", I32, 0), ("frame_y_extent", I32, 8)]
# buffers whose required region the filter checks (-4); every other read clamps or is fixed by a constraint
COVERED = {"halide_blur": ["input"], "local_laplacian": ["input"], SHARDED: ["input"], "bilateral_grid": ["input"],
           "camera_pipe": ["input", "matrix_3200", "matrix_7000"]}
AUTO_SCHEDULED = ["local_laplacian", "bilateral_grid", "nl_means", "stencil_chain", "camera_pipe", "conv_layer"]
METADATA = sorted(list(FILTERS)[:7] + [f + "_auto_schedule" for f in AUTO_SCHEDULED])


def _entries(f):
    """Every entry point that implements filter f: (symbol, called through argv)."""
    if f == SHARDED:
        return [(f, False)]
    names = [f] + ([f + "_auto_schedule"] if f in AUTO_SCHEDULED else [])
    return [(n, False) for n in names] + [(n + "_argv", True) for n in names]


def _is_buffer(spec):
    return len(spec) == 4


_arrays = {}


class Call:
    """One set of arguments for filter f: fresh buffer descriptors over cached host arrays (a checked call never writes
    them), and scalar values, both mutable by a case."""

    def __init__(self, hb, f):
        self.hb, self.f, self.buf, self.val = hb, f, {}, {}
        for spec in FILTERS[f]:
            if _is_buffer(spec):
                name, dtype, shape, mins = spec
                key = (dtype, shape)
                if key not in _arrays:
                    _arrays[key] = np.zeros(shape, dtype)
                self.buf[name] = hb.HalideBuffer.from_numpy(_arrays[key], mins)
            else:
                self.val[spec[0]] = spec[2]

    def dims(self, name):
        return self.buf[name].dims

    def retype(self, name, dtype):
        spec = next(s for s in FILTERS[self.f] if s[0] == name)
        self.buf[name] = self.hb.HalideBuffer.from_numpy(np.zeros(spec[2], dtype), spec[3])

    def query(self, name):
        b = self.buf[name]
        self.buf[name] = self.hb.HalideBuffer.bounds_query(b.dtype, b.buf.dimensions)

    def run(self, symbol, argv):
        fn = getattr(self.hb.load_library(), symbol)
        args = []
        for spec in FILTERS[self.f]:
            if _is_buffer(spec):
                b = self.buf[spec[0]]
                args.append(ctypes.c_void_p(None if b is None else ctypes.addressof(b.buf)))
            else:
                args.append(spec[1](self.val[spec[0]]))
        with self.hb.capture_errors() as err:
            if argv:
                # a buffer slot holds the halide_buffer_t *, a scalar slot the address of the value
                slots = [a.value if isinstance(a, ctypes.c_void_p) else ctypes.addressof(a) for a in args]
                rc = fn((ctypes.c_void_p * len(slots))(*slots))
            else:
                rc = fn(*args)
            return rc, err.msg


def _device_resident(hb, b, interface):
    """Give b a device allocation of `interface` that is current (not host-dirty): acquiring it makes no CUDA call.  The
    address is never dereferenced: every case fails before a launch."""
    b.buf.device = 1 << 40
    b.buf.device_interface = interface
    b.buf.flags = 0


def _forget_device(b):
    b.buf.device, b.buf.device_interface = 0, None


def _buffer_cases(f):
    """(case id, mutate(call)) for the faults every buffer argument can carry."""
    cases = []
    bufs = [s for s in FILTERS[f] if _is_buffer(s)]
    for spec in bufs:
        n, dtype, shape = spec[0], spec[1], spec[2]
        nd = len(shape)
        cases.append((f"{n}/null", lambda c, n=n: c.buf.__setitem__(n, None)))
        cases.append((f"{n}/type", lambda c, n=n, t=(U8 if dtype != U8 else U16): c.retype(n, t)))
        cases.append((f"{n}/dimensions", lambda c, n=n, s=shape: c.buf.__setitem__(
            n, c.hb.HalideBuffer.from_numpy(np.zeros(s + (1,) if len(s) < 4 else s[1:], c.buf[n].dtype)))))
        cases.append((f"{n}/negative_extent", lambda c, n=n, d=nd - 1: setattr(c.dims(n)[d], "extent", -1)))
        cases.append((f"{n}/stride0", lambda c, n=n: setattr(c.dims(n)[0], "stride", 2)))
        cases.append((f"{n}/allocation_too_large", lambda c, n=n, d=nd - 1: setattr(c.dims(n)[d], "stride", 1 << 30)))
        if nd > 1:  # 2^32 elements, each dimension's extent * stride within 2^31 (a zero stride repeats the rows)
            cases.append((f"{n}/extents_too_large", _all(*[lambda c, n=n, d=d, k=k, v=v: setattr(c.dims(n)[d], k, v)
                                                          for d, k, v in [(0, "extent", 1 << 16), (1, "extent", 1 << 16),
                                                                          (1, "stride", 0)]])))
        if f in COVERED and n in COVERED[f]:
            for d in range(nd):
                cases.append((f"{n}/uncovered_min{d}", lambda c, n=n, d=d: setattr(c.dims(n)[d], "min", c.dims(n)[d].min + 1)))
                cases.append((f"{n}/uncovered_max{d}", lambda c, n=n, d=d: setattr(c.dims(n)[d], "extent", c.dims(n)[d].extent - 1)))
    return cases


def _empty(name, d=0):
    return lambda c: setattr(c.dims(name)[d], "extent", 0)


def _set(name, value):
    return lambda c: c.val.__setitem__(name, value)


def _all(*fns):
    def run(c):
        for fn in fns:
            fn(c)
    return run


def _shrink(name, d):
    return lambda c: setattr(c.dims(name)[d], "extent", c.dims(name)[d].extent - 1)


def _filter_cases(f):
    """Scalar and constraint errors of one filter, and pairs of faults that pin the order of its checks."""
    bufs = [s[0] for s in FILTERS[f] if _is_buffer(s)]
    first, out = bufs[0], bufs[-1]
    cases = [
        ("empty_output", _empty(out)),
        # every buffer passes the null/type/dimension checks before any bounds query or shape check
        ("null_first+bad_type_output", _all(lambda c: c.buf.__setitem__(first, None), lambda c: c.retype(out, U8 if c.buf[out].dtype != U8 else U16))),
        ("bad_type_first+null_output", _all(lambda c: c.retype(first, U8 if c.buf[first].dtype != U8 else U16), lambda c: c.buf.__setitem__(out, None))),
        ("query_first+null_output", _all(lambda c: c.query(first), lambda c: c.buf.__setitem__(out, None))),
        # a bounds query returns before the shape checks
        ("query_first+stride0_output", _all(lambda c: c.query(first), lambda c: setattr(c.dims(out)[0], "stride", 2))),
        ("stride0_first+negative_extent_output", _all(lambda c: setattr(c.dims(first)[0], "stride", 2),
                                                      lambda c: setattr(c.dims(out)[0], "extent", -1))),
    ]
    ll = [("levels_1", _set("levels", 1)), ("levels_33", _set("levels", 33)),
          ("uncovered_input+levels_1", _all(_shrink("input", 1), _set("levels", 1))),
          ("levels_1+empty_output", _all(_set("levels", 1), _empty("output", 1))),
          ("empty_channels+levels_1", _all(_empty("output", 2), _set("levels", 1)))]
    cases += {
        "halide_blur": [("empty_output+uncovered_input", _all(_empty("blur_y"), _shrink("input", 1))),
                        ("empty_output_rows", _empty("blur_y", 1))],
        "local_laplacian": ll,
        SHARDED: ll + [("no_communicator", lambda c: None), ("empty_output+no_communicator", _empty("output", 1))],
        "bilateral_grid": [("r_sigma_0", _set("r_sigma", 0.0)), ("r_sigma_negative", _set("r_sigma", -1.0)),
                           ("r_sigma_nan", _set("r_sigma", float("nan"))), ("r_sigma_too_many_bins", _set("r_sigma", 0.001)),
                           ("uncovered_input+empty_output", _all(_shrink("input", 1), _empty("bilateral_grid"))),
                           ("empty_output+r_sigma_0", _all(_empty("bilateral_grid"), _set("r_sigma", 0.0))),
                           ("r_sigma_0+r_sigma_bins", _set("r_sigma", -0.001))],
        "nl_means": [("output_channels_4", lambda c: setattr(c.dims("non_local_means")[2], "extent", 4)),
                     ("output_channel_min_1", lambda c: setattr(c.dims("non_local_means")[2], "min", 1)),
                     ("empty_input", _empty("input", 1)),
                     ("patch_0", _set("patch_size", 0)), ("search_0", _set("search_area", 0)),
                     ("patch_32", _set("patch_size", 32)), ("search_64", _set("search_area", 64)),
                     ("patch_0+search_64", _all(_set("patch_size", 0), _set("search_area", 64))),
                     ("output_channels_4+empty_output", _all(lambda c: setattr(c.dims("non_local_means")[2], "extent", 4),
                                                              _empty("non_local_means"))),
                     ("empty_output+empty_input", _all(_empty("non_local_means"), _empty("input"))),
                     ("empty_input+patch_0", _all(_empty("input", 2), _set("patch_size", 0)))],
        "stencil_chain": [("empty_input", _empty("input", 1)),
                          ("empty_output+empty_input", _all(_empty("output", 1), _empty("input")))],
        "camera_pipe": [("empty_channels", _empty("processed", 2)),
                        ("empty_output+uncovered_input", _all(_empty("processed"), _shrink("input", 0))),
                        ("empty_channels+uncovered_matrix", _all(_empty("processed", 2), _shrink("matrix_7000", 0))),
                        ("channels_4", lambda c: setattr(c.dims("processed")[2], "extent", 4)),
                        ("channel_min_1", lambda c: setattr(c.dims("processed")[2], "min", 1)),
                        ("channel_min_negative", lambda c: setattr(c.dims("processed")[2], "min", -1)),
                        ("channels_4+uncovered_input", _all(lambda c: setattr(c.dims("processed")[2], "extent", 4),
                                                            _shrink("input", 1)))],
        "conv_layer": [(f"{n}_{what}", lambda c, n=n, d=d, field=field, v=v: setattr(c.dims(n)[d], field, v))
                       for n, d, field, v, what in [("relu", 3, "extent", 4, "extent3"), ("input", 1, "extent", 81, "extent1"),
                                                    ("filter", 0, "min", 1, "min0"), ("bias", 0, "extent", 64, "extent0"),
                                                    ("input", 2, "stride", 82 * 128 + 1, "stride2"),
                                                    ("relu", 0, "min", -1, "min0")]] +
                      [("relu_extent+input_extent", _all(lambda c: setattr(c.dims("relu")[1], "extent", 99),
                                                         lambda c: setattr(c.dims("input")[1], "extent", 101))),
                       ("bias_extent+filter_extent", _all(lambda c: setattr(c.dims("bias")[0], "extent", 64),
                                                          lambda c: setattr(c.dims("filter")[3], "extent", 64)))],
    }[f]
    return cases


def _cases(f):
    """(case id, mutate(call), foreign, before).  `foreign` names a buffer that already has a device allocation of another
    device interface; the buffers acquired before it (`before`) are made current device allocations of this library, so
    that acquiring them makes no CUDA call."""
    bufs = [s[0] for s in FILTERS[f] if _is_buffer(s)]
    return [(cid, fn, None, []) for cid, fn in _buffer_cases(f) + _filter_cases(f)] + \
           [(f"{n}/foreign_device", None, n, bufs[:i]) for i, n in enumerate(bufs)]


def _run_case(hb, f, symbol, argv, fn, foreign, before):
    c = Call(hb, f)
    if foreign is None:
        fn(c)
        return c.run(symbol, argv)
    ours = hb.capi.halide_cuda_device_interface()
    other = ctypes.create_string_buffer(128)
    for n in before:
        _device_resident(hb, c.buf[n], ours)
    _device_resident(hb, c.buf[foreign], ctypes.addressof(other))
    try:
        return c.run(symbol, argv)
    finally:
        for n in before + [foreign]:
            _forget_device(c.buf[n])


@pytest.mark.parametrize("f", list(FILTERS))
def test_argument_errors(hb, f):
    want = ERRORS[f]
    got = {}
    for cid, fn, foreign, before in _cases(f):
        for symbol, argv in _entries(f):
            r = _run_case(hb, f, symbol, argv, fn, foreign, before)
            assert got.setdefault(cid, r) == r, (cid, symbol, r, got[cid])
    assert got == want


def _query_shapes(c, names):
    return {n: [tuple(t) for t in c.buf[n].shape()] for n in names}


@pytest.mark.parametrize("f", list(FILTERS))
def test_bounds_queries(hb, f):
    bufs = [s[0] for s in FILTERS[f] if _is_buffer(s)]
    got = {}
    for queried in [[n] for n in bufs] + [bufs]:
        for symbol, argv in _entries(f):
            c = Call(hb, f)
            for n in queried:
                c.query(n)
            r = (c.run(symbol, argv), _query_shapes(c, queried))
            key = "+".join(queried)
            assert got.setdefault(key, r) == r, (key, symbol, r, got[key])
    assert got == QUERIES[f]


class _Meta(ctypes.Structure):
    _fields_ = [("version", ctypes.c_int32), ("num_arguments", ctypes.c_int32), ("arguments", ctypes.c_void_p),
                ("target", ctypes.c_char_p), ("name", ctypes.c_char_p)]


class _Arg(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char_p), ("kind", ctypes.c_int32), ("dimensions", ctypes.c_int32),
                ("code", ctypes.c_uint8), ("bits", ctypes.c_uint8), ("lanes", ctypes.c_uint16),
                ("scalar_def", ctypes.c_void_p), ("scalar_min", ctypes.c_void_p), ("scalar_max", ctypes.c_void_p),
                ("scalar_estimate", ctypes.c_void_p), ("buffer_estimates", ctypes.POINTER(ctypes.POINTER(ctypes.c_int64)))]


def _scalar(p):
    return None if not p else ctypes.string_at(p, 8).hex()


def _metadata(hb, symbol):
    fn = getattr(hb.load_library(), symbol + "_metadata")
    fn.restype = ctypes.POINTER(_Meta)
    m = fn().contents
    args = []
    for a in (_Arg * m.num_arguments).from_address(m.arguments):
        est = None
        if a.buffer_estimates:
            est = [None if not a.buffer_estimates[i] else a.buffer_estimates[i][0] for i in range(2 * a.dimensions)]
        args.append((a.name.decode(), a.kind, a.dimensions, (a.code, a.bits, a.lanes), _scalar(a.scalar_def), _scalar(a.scalar_min),
                     _scalar(a.scalar_max), _scalar(a.scalar_estimate), est))
    return m.version, m.num_arguments, m.name.decode(), m.target.decode(), args


@pytest.mark.parametrize("symbol", METADATA)
def test_metadata(hb, symbol):
    version, n, name, target, args = _metadata(hb, symbol)
    assert name == symbol
    assert target == hb.capi.halide_b200_target().decode() == TARGET
    assert (version, n, args) == METADATA_RECORDS[symbol.removesuffix("_auto_schedule")]


def _inputs(f, rng):
    """Seeded contents for each input buffer of filter f (the valid shapes above), chosen so that the filter does real
    work."""
    data = {}
    for n, dtype, shape, _ in [s for s in FILTERS[f] if _is_buffer(s)][:-1]:
        if dtype == F32:
            data[n] = rng.random(shape, dtype=np.float32)
        else:
            data[n] = rng.integers(0, 1024 if f == "camera_pipe" else np.iinfo(dtype).max, shape, dtype=dtype)
    if f == "camera_pipe":
        for m in ("matrix_3200", "matrix_7000"):
            data[m] = (np.eye(3, 4, dtype=np.float32) + 0.05 * data[m]).astype(np.float32)
    return data


# scalars that differ from the valid defaults above, so a mix-up between argv slots changes the result
GPU_SCALARS = {
    "local_laplacian": {"levels": 6, "alpha": 0.3, "beta": 1.4},
    "bilateral_grid": {"r_sigma": 0.2},
    "nl_means": {"patch_size": 5, "search_area": 5, "sigma": 0.3},
    "camera_pipe": {"color_temp": 4200.0, "gamma": 1.8, "contrast": 30.0, "sharpen_strength": 0.5, "blackLevel": 20, "whiteLevel": 1000},
}


@pytest.mark.gpu
@pytest.mark.parametrize("f", list(FILTERS)[:7])
def test_entry_points_compute_the_same(hb, f):
    data = _inputs(f, np.random.default_rng(7))
    out, dtype, shape, mins = [s for s in FILTERS[f] if _is_buffer(s)][-1]
    results = {}
    for symbol, argv in _entries(f):
        c = Call(hb, f)
        for n, a in data.items():
            c.buf[n] = hb.HalideBuffer.from_numpy(a, [d[0] for d in c.buf[n].shape()])
        dst = np.zeros(shape, dtype)
        c.buf[out] = hb.HalideBuffer.from_numpy(dst, mins, host_dirty=False)
        c.val.update(GPU_SCALARS.get(f, {}))
        assert c.run(symbol, argv) == (0, "")
        c.buf[out].copy_to_host()
        results[symbol] = dst
    first = results[f]
    assert first.any()
    for symbol, r in results.items():
        assert r.tobytes() == first.tobytes(), symbol


# ---- expected values, captured from the library ----
TARGET = "x86-64-linux-cuda-cuda_capability_90-h100_native"
# per filter (F_metadata and F_auto_schedule_metadata): version, num_arguments, and per argument: name, kind,
# dimensions, type (code, bits, lanes), the 8 bytes of scalar def/min/max/estimate (hex), buffer estimates
METADATA_RECORDS = {
    "bilateral_grid": (1, 3, [
        ("input", 1, 2, (2, 32, 0), None, None, None, None, [0, 1536, 0, 2560]),
        ("r_sigma", 0, 0, (2, 32, 0), None, None, None, "cdcccc3d00000000", None),
        ("bilateral_grid", 2, 2, (2, 32, 0), None, None, None, None, [0, 1536, 0, 2560]),
    ]),
    "camera_pipe": (1, 10, [
        ("input", 1, 2, (1, 16, 0), None, None, None, None, [0, 2592, 0, 1968]),
        ("matrix_3200", 1, 2, (2, 32, 0), None, None, None, None, [0, 4, 0, 3]),
        ("matrix_7000", 1, 2, (2, 32, 0), None, None, None, None, [0, 4, 0, 3]),
        ("color_temp", 0, 0, (2, 32, 0), None, None, None, "0040674500000000", None),
        ("gamma", 0, 0, (2, 32, 0), None, None, None, "0000004000000000", None),
        ("contrast", 0, 0, (2, 32, 0), None, None, None, "0000484200000000", None),
        ("sharpen_strength", 0, 0, (2, 32, 0), None, None, None, "0000803f00000000", None),
        ("blackLevel", 0, 0, (0, 32, 0), None, None, None, "1900000000000000", None),
        ("whiteLevel", 0, 0, (0, 32, 0), None, None, None, "ff03000000000000", None),
        ("processed", 2, 3, (1, 8, 0), None, None, None, None, [0, 2592, 0, 1968, 0, 3]),
    ]),
    "conv_layer": (1, 4, [
        ("input", 1, 4, (2, 32, 0), None, None, None, None, [0, 128, 0, 102, 0, 82, 0, 5]),
        ("filter", 1, 4, (2, 32, 0), None, None, None, None, [0, 128, 0, 3, 0, 3, 0, 128]),
        ("bias", 1, 1, (2, 32, 0), None, None, None, None, [0, 128]),
        ("relu", 2, 4, (2, 32, 0), None, None, None, None, [0, 128, 0, 100, 0, 80, 0, 5]),
    ]),
    "halide_blur": (1, 2, [
        ("input", 1, 2, (1, 16, 0), None, None, None, None, None),
        ("blur_y", 2, 2, (1, 16, 0), None, None, None, None, None),
    ]),
    "local_laplacian": (1, 5, [
        ("input", 1, 3, (1, 16, 0), None, None, None, None, [0, 1536, 0, 2560, 0, 3]),
        ("levels", 0, 0, (0, 32, 0), None, None, None, "0800000000000000", None),
        ("alpha", 0, 0, (2, 32, 0), None, None, None, "0000803f00000000", None),
        ("beta", 0, 0, (2, 32, 0), None, None, None, "0000803f00000000", None),
        ("output", 2, 3, (1, 16, 0), None, None, None, None, [0, 1536, 0, 2560, 0, 3]),
    ]),
    "nl_means": (1, 5, [
        ("input", 1, 3, (2, 32, 0), None, None, None, None, [0, 1536, 0, 2560, 0, 3]),
        ("patch_size", 0, 0, (0, 32, 0), None, None, None, "0700000000000000", None),
        ("search_area", 0, 0, (0, 32, 0), None, None, None, "0700000000000000", None),
        ("sigma", 0, 0, (2, 32, 0), None, None, None, "8fc2f53d00000000", None),
        ("non_local_means", 2, 3, (2, 32, 0), None, None, None, None, [0, 1536, 0, 2560, 0, 3]),
    ]),
    "stencil_chain": (1, 2, [
        ("input", 1, 2, (1, 16, 0), None, None, None, None, [0, 1536, 0, 2560]),
        ("output", 2, 2, (1, 16, 0), None, None, None, None, [0, 1536, 0, 2560]),
    ]),
}
# per filter and case: (return code, halide_error message)
ERRORS = {
    "halide_blur": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 1 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 12884901888, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "input/uncovered_min0": (-4, "Input buffer input is accessed at 2, which is before the min (3) in dimension 0"),
        "input/uncovered_max0": (-4, "Input buffer input is accessed at 19, which is beyond the max (18) in dimension 0"),
        "input/uncovered_min1": (-4, "Input buffer input is accessed at 3, which is before the min (4) in dimension 1"),
        "input/uncovered_max1": (-4, "Input buffer input is accessed at 14, which is beyond the max (13) in dimension 1"),
        "blur_y/null": (-12, "Buffer argument blur_y is nullptr"),
        "blur_y/type": (-3, "Output buffer blur_y has type code 1 bits 8 but expected code 1 bits 16"),
        "blur_y/dimensions": (-43, "Output buffer blur_y requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "blur_y/negative_extent": (-28, "The extents for buffer blur_y dimension 1 is negative (-1)"),
        "blur_y/stride0": (-8, "Constraint violated: blur_y.stride.0 (2) == 1 (1)"),
        "blur_y/allocation_too_large": (-5, "Total allocation for buffer blur_y is 10737418240, which exceeds the maximum size of 2147483647"),
        "blur_y/extents_too_large": (-6, "Product of extents for buffer blur_y is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "query_first+null_output": (-12, "Buffer argument blur_y is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "empty_output+uncovered_input": (-4, "Input buffer input is accessed at 14, which is beyond the max (13) in dimension 1"),
        "empty_output_rows": (0, ""),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "blur_y/foreign_device": (-42, "Output buffer blur_y has a device allocation of a different device interface"),
    },
    "local_laplacian": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 2 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 3221225472, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "input/uncovered_min0": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 0"),
        "input/uncovered_max0": (-4, "Input buffer input is accessed at 9, which is beyond the max (8) in dimension 0"),
        "input/uncovered_min1": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 1"),
        "input/uncovered_max1": (-4, "Input buffer input is accessed at 7, which is beyond the max (6) in dimension 1"),
        "input/uncovered_min2": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 2"),
        "input/uncovered_max2": (-4, "Input buffer input is accessed at 2, which is beyond the max (1) in dimension 2"),
        "output/null": (-12, "Buffer argument output is nullptr"),
        "output/type": (-3, "Output buffer output has type code 1 bits 8 but expected code 1 bits 16"),
        "output/dimensions": (-43, "Output buffer output requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "output/negative_extent": (-28, "The extents for buffer output dimension 2 is negative (-1)"),
        "output/stride0": (-8, "Constraint violated: output.stride.0 (2) == 1 (1)"),
        "output/allocation_too_large": (-5, "Total allocation for buffer output is 3221225472, which exceeds the maximum size of 2147483647"),
        "output/extents_too_large": (-6, "Product of extents for buffer output is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "query_first+null_output": (-12, "Buffer argument output is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "levels_1": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "levels_33": (-10, "Parameter levels is 33 but must be in [2, 32]"),
        "uncovered_input+levels_1": (-4, "Input buffer input is accessed at 7, which is beyond the max (6) in dimension 1"),
        "levels_1+empty_output": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "empty_channels+levels_1": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "output/foreign_device": (-42, "Output buffer output has a device allocation of a different device interface"),
    },
    "bilateral_grid": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 1 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 8589934592, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "input/uncovered_min0": (-4, "Input buffer input is accessed at 1, which is before the min (2) in dimension 0"),
        "input/uncovered_max0": (-4, "Input buffer input is accessed at 10, which is beyond the max (9) in dimension 0"),
        "input/uncovered_min1": (-4, "Input buffer input is accessed at 2, which is before the min (3) in dimension 1"),
        "input/uncovered_max1": (-4, "Input buffer input is accessed at 9, which is beyond the max (8) in dimension 1"),
        "bilateral_grid/null": (-12, "Buffer argument bilateral_grid is nullptr"),
        "bilateral_grid/type": (-3, "Output buffer bilateral_grid has type code 1 bits 8 but expected code 2 bits 32"),
        "bilateral_grid/dimensions": (-43, "Output buffer bilateral_grid requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "bilateral_grid/negative_extent": (-28, "The extents for buffer bilateral_grid dimension 1 is negative (-1)"),
        "bilateral_grid/stride0": (-8, "Constraint violated: bilateral_grid.stride.0 (2) == 1 (1)"),
        "bilateral_grid/allocation_too_large": (-5, "Total allocation for buffer bilateral_grid is 8589934592, which exceeds the maximum size of 2147483647"),
        "bilateral_grid/extents_too_large": (-6, "Product of extents for buffer bilateral_grid is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "query_first+null_output": (-12, "Buffer argument bilateral_grid is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "r_sigma_0": (-9, "Parameter r_sigma is 0 but must be positive"),
        "r_sigma_negative": (-9, "Parameter r_sigma is -1 but must be positive"),
        "r_sigma_nan": (-9, "Parameter r_sigma is nan but must be positive"),
        "r_sigma_too_many_bins": (-9, "Parameter r_sigma is 0.001: more than 200 intensity bins are not supported by this build"),
        "uncovered_input+empty_output": (-4, "Input buffer input is accessed at 9, which is beyond the max (8) in dimension 1"),
        "empty_output+r_sigma_0": (0, ""),
        "r_sigma_0+r_sigma_bins": (-9, "Parameter r_sigma is -0.001 but must be positive"),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "bilateral_grid/foreign_device": (-42, "Output buffer bilateral_grid has a device allocation of a different device interface"),
    },
    "nl_means": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 2 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 3221225472, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "non_local_means/null": (-12, "Buffer argument non_local_means is nullptr"),
        "non_local_means/type": (-3, "Output buffer non_local_means has type code 1 bits 8 but expected code 2 bits 32"),
        "non_local_means/dimensions": (-43, "Output buffer non_local_means requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "non_local_means/negative_extent": (-28, "The extents for buffer non_local_means dimension 2 is negative (-1)"),
        "non_local_means/stride0": (-8, "Constraint violated: non_local_means.stride.0 (2) == 1 (1)"),
        "non_local_means/allocation_too_large": (-5, "Total allocation for buffer non_local_means is 3221225472, which exceeds the maximum size of 2147483647"),
        "non_local_means/extents_too_large": (-6, "Product of extents for buffer non_local_means is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "query_first+null_output": (-12, "Buffer argument non_local_means is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "output_channels_4": (-8, "Constraint violated: non_local_means.min.2 (0) == 0 and non_local_means.extent.2 (4) == 3"),
        "output_channel_min_1": (-8, "Constraint violated: non_local_means.min.2 (1) == 0 and non_local_means.extent.2 (3) == 3"),
        "empty_input": (-4, "Input buffer input is empty"),
        "patch_0": (-9, "nl_means: patch_size 0 / search_area 7 outside the supported range [1,31] / [1,63]"),
        "search_0": (-9, "nl_means: patch_size 3 / search_area 0 outside the supported range [1,31] / [1,63]"),
        "patch_32": (-10, "nl_means: patch_size 32 / search_area 7 outside the supported range [1,31] / [1,63]"),
        "search_64": (-10, "nl_means: patch_size 3 / search_area 64 outside the supported range [1,31] / [1,63]"),
        "patch_0+search_64": (-9, "nl_means: patch_size 0 / search_area 64 outside the supported range [1,31] / [1,63]"),
        "output_channels_4+empty_output": (-8, "Constraint violated: non_local_means.min.2 (0) == 0 and non_local_means.extent.2 (4) == 3"),
        "empty_output+empty_input": (0, ""),
        "empty_input+patch_0": (-4, "Input buffer input is empty"),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "non_local_means/foreign_device": (-42, "Output buffer non_local_means has a device allocation of a different device interface"),
    },
    "stencil_chain": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 1 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 8589934592, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "output/null": (-12, "Buffer argument output is nullptr"),
        "output/type": (-3, "Output buffer output has type code 1 bits 8 but expected code 1 bits 16"),
        "output/dimensions": (-43, "Output buffer output requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "output/negative_extent": (-28, "The extents for buffer output dimension 1 is negative (-1)"),
        "output/stride0": (-8, "Constraint violated: output.stride.0 (2) == 1 (1)"),
        "output/allocation_too_large": (-5, "Total allocation for buffer output is 8589934592, which exceeds the maximum size of 2147483647"),
        "output/extents_too_large": (-6, "Product of extents for buffer output is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "query_first+null_output": (-12, "Buffer argument output is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "empty_input": (-4, "Input buffer input is empty"),
        "empty_output+empty_input": (0, ""),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "output/foreign_device": (-42, "Output buffer output has a device allocation of a different device interface"),
    },
    "camera_pipe": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 1 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 47244640256, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "input/uncovered_min0": (-4, "Input buffer input is accessed at 10, which is before the min (11) in dimension 0"),
        "input/uncovered_max0": (-4, "Input buffer input is accessed at 61, which is beyond the max (60) in dimension 0"),
        "input/uncovered_min1": (-4, "Input buffer input is accessed at 6, which is before the min (7) in dimension 1"),
        "input/uncovered_max1": (-4, "Input buffer input is accessed at 49, which is beyond the max (48) in dimension 1"),
        "matrix_3200/null": (-12, "Buffer argument matrix_3200 is nullptr"),
        "matrix_3200/type": (-3, "Input buffer matrix_3200 has type code 1 bits 8 but expected code 2 bits 32"),
        "matrix_3200/dimensions": (-43, "Input buffer matrix_3200 requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "matrix_3200/negative_extent": (-28, "The extents for buffer matrix_3200 dimension 1 is negative (-1)"),
        "matrix_3200/stride0": (-8, "Constraint violated: matrix_3200.stride.0 (2) == 1 (1)"),
        "matrix_3200/allocation_too_large": (-5, "Total allocation for buffer matrix_3200 is 3221225472, which exceeds the maximum size of 2147483647"),
        "matrix_3200/extents_too_large": (-6, "Product of extents for buffer matrix_3200 is 4294967296, which exceeds the maximum size of 2147483647"),
        "matrix_3200/uncovered_min0": (-4, "Input buffer matrix_3200 is accessed at 0, which is before the min (1) in dimension 0"),
        "matrix_3200/uncovered_max0": (-4, "Input buffer matrix_3200 is accessed at 3, which is beyond the max (2) in dimension 0"),
        "matrix_3200/uncovered_min1": (-4, "Input buffer matrix_3200 is accessed at 0, which is before the min (1) in dimension 1"),
        "matrix_3200/uncovered_max1": (-4, "Input buffer matrix_3200 is accessed at 2, which is beyond the max (1) in dimension 1"),
        "matrix_7000/null": (-12, "Buffer argument matrix_7000 is nullptr"),
        "matrix_7000/type": (-3, "Input buffer matrix_7000 has type code 1 bits 8 but expected code 2 bits 32"),
        "matrix_7000/dimensions": (-43, "Input buffer matrix_7000 requires a buffer of exactly 2 dimensions, but the buffer passed in has 3 dimensions"),
        "matrix_7000/negative_extent": (-28, "The extents for buffer matrix_7000 dimension 1 is negative (-1)"),
        "matrix_7000/stride0": (-8, "Constraint violated: matrix_7000.stride.0 (2) == 1 (1)"),
        "matrix_7000/allocation_too_large": (-5, "Total allocation for buffer matrix_7000 is 3221225472, which exceeds the maximum size of 2147483647"),
        "matrix_7000/extents_too_large": (-6, "Product of extents for buffer matrix_7000 is 4294967296, which exceeds the maximum size of 2147483647"),
        "matrix_7000/uncovered_min0": (-4, "Input buffer matrix_7000 is accessed at 0, which is before the min (1) in dimension 0"),
        "matrix_7000/uncovered_max0": (-4, "Input buffer matrix_7000 is accessed at 3, which is beyond the max (2) in dimension 0"),
        "matrix_7000/uncovered_min1": (-4, "Input buffer matrix_7000 is accessed at 0, which is before the min (1) in dimension 1"),
        "matrix_7000/uncovered_max1": (-4, "Input buffer matrix_7000 is accessed at 2, which is beyond the max (1) in dimension 1"),
        "processed/null": (-12, "Buffer argument processed is nullptr"),
        "processed/type": (-3, "Output buffer processed has type code 1 bits 16 but expected code 1 bits 8"),
        "processed/dimensions": (-43, "Output buffer processed requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "processed/negative_extent": (-28, "The extents for buffer processed dimension 2 is negative (-1)"),
        "processed/stride0": (-8, "Constraint violated: processed.stride.0 (2) == 1 (1)"),
        "processed/allocation_too_large": (-5, "Total allocation for buffer processed is 3221225472, which exceeds the maximum size of 2147483647"),
        "processed/extents_too_large": (-6, "Product of extents for buffer processed is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "query_first+null_output": (-12, "Buffer argument processed is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "empty_channels": (0, ""),
        "empty_output+uncovered_input": (0, ""),
        "empty_channels+uncovered_matrix": (0, ""),
        "channels_4": (-4, "Output buffer processed channel range [0,4) is outside [0,3)"),
        "channel_min_1": (-4, "Output buffer processed channel range [1,4) is outside [0,3)"),
        "channel_min_negative": (-4, "Output buffer processed channel range [-1,2) is outside [0,3)"),
        "channels_4+uncovered_input": (-4, "Input buffer input is accessed at 49, which is beyond the max (48) in dimension 1"),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "matrix_3200/foreign_device": (-42, "Input buffer matrix_3200 has a device allocation of a different device interface"),
        "matrix_7000/foreign_device": (-42, "Input buffer matrix_7000 has a device allocation of a different device interface"),
        "processed/foreign_device": (-42, "Output buffer processed has a device allocation of a different device interface"),
    },
    "conv_layer": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 4 dimensions, but the buffer passed in has 3 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 3 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 5368709120, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "filter/null": (-12, "Buffer argument filter is nullptr"),
        "filter/type": (-3, "Input buffer filter has type code 1 bits 8 but expected code 2 bits 32"),
        "filter/dimensions": (-43, "Input buffer filter requires a buffer of exactly 4 dimensions, but the buffer passed in has 3 dimensions"),
        "filter/negative_extent": (-28, "The extents for buffer filter dimension 3 is negative (-1)"),
        "filter/stride0": (-8, "Constraint violated: filter.stride.0 (2) == 1 (1)"),
        "filter/allocation_too_large": (-5, "Total allocation for buffer filter is 137438953472, which exceeds the maximum size of 2147483647"),
        "filter/extents_too_large": (-6, "Product of extents for buffer filter is 4294967296, which exceeds the maximum size of 2147483647"),
        "bias/null": (-12, "Buffer argument bias is nullptr"),
        "bias/type": (-3, "Input buffer bias has type code 1 bits 8 but expected code 2 bits 32"),
        "bias/dimensions": (-43, "Input buffer bias requires a buffer of exactly 1 dimensions, but the buffer passed in has 2 dimensions"),
        "bias/negative_extent": (-28, "The extents for buffer bias dimension 0 is negative (-1)"),
        "bias/stride0": (-8, "Constraint violated: bias.stride.0 (2) == 1 (1)"),
        "bias/allocation_too_large": (-5, "Total allocation for buffer bias is 137438953472, which exceeds the maximum size of 2147483647"),
        "relu/null": (-12, "Buffer argument relu is nullptr"),
        "relu/type": (-3, "Output buffer relu has type code 1 bits 8 but expected code 2 bits 32"),
        "relu/dimensions": (-43, "Output buffer relu requires a buffer of exactly 4 dimensions, but the buffer passed in has 3 dimensions"),
        "relu/negative_extent": (-28, "The extents for buffer relu dimension 3 is negative (-1)"),
        "relu/stride0": (-8, "Constraint violated: relu.stride.0 (2) == 1 (1)"),
        "relu/allocation_too_large": (-5, "Total allocation for buffer relu is 5368709120, which exceeds the maximum size of 2147483647"),
        "relu/extents_too_large": (-6, "Product of extents for buffer relu is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (-8, "Constraint violated: relu.dim(0) is (min 0, extent 0, stride 1) but must be (0, 128, 1)"),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 2 bits 32"),
        "query_first+null_output": (-12, "Buffer argument relu is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "relu_extent3": (-8, "Constraint violated: relu.dim(3) is (min 0, extent 4, stride 1024000) but must be (0, 5, 1024000)"),
        "input_extent1": (-8, "Constraint violated: input.dim(1) is (min 0, extent 81, stride 128) but must be (0, 102, 128)"),
        "filter_min0": (-8, "Constraint violated: filter.dim(0) is (min 1, extent 128, stride 1) but must be (0, 128, 1)"),
        "bias_extent0": (-8, "Constraint violated: bias.dim(0) is (min 0, extent 64, stride 1) but must be (0, 128, 1)"),
        "input_stride2": (-8, "Constraint violated: input.dim(2) is (min 0, extent 82, stride 10497) but must be (0, 82, 13056)"),
        "relu_min0": (-8, "Constraint violated: relu.dim(0) is (min -1, extent 128, stride 1) but must be (0, 128, 1)"),
        "relu_extent+input_extent": (-8, "Constraint violated: relu.dim(1) is (min 0, extent 99, stride 128) but must be (0, 100, 128)"),
        "bias_extent+filter_extent": (-8, "Constraint violated: filter.dim(3) is (min 0, extent 64, stride 1152) but must be (0, 128, 1152)"),
        "input/foreign_device": (-42, "Input buffer input has a device allocation of a different device interface"),
        "filter/foreign_device": (-42, "Input buffer filter has a device allocation of a different device interface"),
        "bias/foreign_device": (-42, "Input buffer bias has a device allocation of a different device interface"),
        "relu/foreign_device": (-42, "Output buffer relu has a device allocation of a different device interface"),
    },
    "halide_b200_local_laplacian_sharded": {
        "input/null": (-12, "Buffer argument input is nullptr"),
        "input/type": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "input/dimensions": (-43, "Input buffer input requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "input/negative_extent": (-28, "The extents for buffer input dimension 2 is negative (-1)"),
        "input/stride0": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "input/allocation_too_large": (-5, "Total allocation for buffer input is 3221225472, which exceeds the maximum size of 2147483647"),
        "input/extents_too_large": (-6, "Product of extents for buffer input is 4294967296, which exceeds the maximum size of 2147483647"),
        "input/uncovered_min0": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 0"),
        "input/uncovered_max0": (-4, "Input buffer input is accessed at 9, which is beyond the max (8) in dimension 0"),
        "input/uncovered_min1": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 1"),
        "input/uncovered_max1": (-4, "Input buffer input is accessed at 7, which is beyond the max (6) in dimension 1"),
        "input/uncovered_min2": (-4, "Input buffer input is accessed at 0, which is before the min (1) in dimension 2"),
        "input/uncovered_max2": (-4, "Input buffer input is accessed at 2, which is beyond the max (1) in dimension 2"),
        "output/null": (-12, "Buffer argument output is nullptr"),
        "output/type": (-3, "Output buffer output has type code 1 bits 8 but expected code 1 bits 16"),
        "output/dimensions": (-43, "Output buffer output requires a buffer of exactly 3 dimensions, but the buffer passed in has 4 dimensions"),
        "output/negative_extent": (-28, "The extents for buffer output dimension 2 is negative (-1)"),
        "output/stride0": (-8, "Constraint violated: output.stride.0 (2) == 1 (1)"),
        "output/allocation_too_large": (-5, "Total allocation for buffer output is 3221225472, which exceeds the maximum size of 2147483647"),
        "output/extents_too_large": (-6, "Product of extents for buffer output is 4294967296, which exceeds the maximum size of 2147483647"),
        "empty_output": (0, ""),
        "null_first+bad_type_output": (-12, "Buffer argument input is nullptr"),
        "bad_type_first+null_output": (-3, "Input buffer input has type code 1 bits 8 but expected code 1 bits 16"),
        "query_first+null_output": (-12, "Buffer argument output is nullptr"),
        "query_first+stride0_output": (0, ""),
        "stride0_first+negative_extent_output": (-8, "Constraint violated: input.stride.0 (2) == 1 (1)"),
        "levels_1": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "levels_33": (-10, "Parameter levels is 33 but must be in [2, 32]"),
        "uncovered_input+levels_1": (-4, "Input buffer input is accessed at 7, which is beyond the max (6) in dimension 1"),
        "levels_1+empty_output": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "empty_channels+levels_1": (-9, "Parameter levels is 1 but must be in [2, 32]"),
        "no_communicator": (-1, "local_laplacian_sharded: call halide_b200_dist_init first"),
        "empty_output+no_communicator": (0, ""),
        "input/foreign_device": (-1, "local_laplacian_sharded: call halide_b200_dist_init first"),
        "output/foreign_device": (-1, "local_laplacian_sharded: call halide_b200_dist_init first"),
    },
}
# per filter and set of queried buffers: ((return code, message), {buffer: [(min, extent, stride) per dimension]})
QUERIES = {
    "halide_blur": {
        "input": ((0, ""), {"input": [(2, 18, 1), (3, 12, 18)]}),
        "blur_y": ((0, ""), {"blur_y": [(0, 0, 1), (0, 0, 0)]}),
        "input+blur_y": ((0, ""), {"input": [(0, 2, 1), (0, 2, 2)], "blur_y": [(0, 0, 1), (0, 0, 0)]}),
    },
    "local_laplacian": {
        "input": ((0, ""), {"input": [(0, 10, 1), (0, 8, 10), (0, 3, 80)]}),
        "output": ((0, ""), {"output": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
        "input+output": ((0, ""), {"input": [(0, 0, 1), (0, 0, 0), (0, 0, 0)], "output": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
    },
    "bilateral_grid": {
        "input": ((0, ""), {"input": [(1, 10, 1), (2, 8, 10)]}),
        "bilateral_grid": ((0, ""), {"bilateral_grid": [(0, 0, 1), (0, 0, 0)]}),
        "input+bilateral_grid": ((0, ""), {"input": [(0, 0, 1), (0, 0, 0)], "bilateral_grid": [(0, 0, 1), (0, 0, 0)]}),
    },
    "nl_means": {
        "input": ((0, ""), {"input": [(0, 10, 1), (0, 8, 10), (0, 3, 80)]}),
        "non_local_means": ((0, ""), {"non_local_means": [(0, 0, 1), (0, 0, 0), (0, 3, 0)]}),
        "input+non_local_means": ((0, ""), {"input": [(0, 0, 1), (0, 0, 0), (0, 3, 0)], "non_local_means": [(0, 0, 1), (0, 0, 0), (0, 3, 0)]}),
    },
    "stencil_chain": {
        "input": ((0, ""), {"input": [(0, 10, 1), (0, 8, 10)]}),
        "output": ((0, ""), {"output": [(0, 0, 1), (0, 0, 0)]}),
        "input+output": ((0, ""), {"input": [(0, 0, 1), (0, 0, 0)], "output": [(0, 0, 1), (0, 0, 0)]}),
    },
    "camera_pipe": {
        "input": ((0, ""), {"input": [(10, 52, 1), (6, 44, 52)]}),
        "matrix_3200": ((0, ""), {"matrix_3200": [(0, 4, 1), (0, 3, 4)]}),
        "matrix_7000": ((0, ""), {"matrix_7000": [(0, 4, 1), (0, 3, 4)]}),
        "processed": ((0, ""), {"processed": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
        "input+matrix_3200+matrix_7000+processed": ((0, ""), {"input": [(10, 12, 1), (6, 12, 12)], "matrix_3200": [(0, 4, 1), (0, 3, 4)], "matrix_7000": [(0, 4, 1), (0, 3, 4)], "processed": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
    },
    "conv_layer": {
        "input": ((0, ""), {"input": [(0, 128, 1), (0, 102, 128), (0, 82, 13056), (0, 5, 1070592)]}),
        "filter": ((0, ""), {"filter": [(0, 128, 1), (0, 3, 128), (0, 3, 384), (0, 128, 1152)]}),
        "bias": ((0, ""), {"bias": [(0, 128, 1)]}),
        "relu": ((0, ""), {"relu": [(0, 128, 1), (0, 100, 128), (0, 80, 12800), (0, 5, 1024000)]}),
        "input+filter+bias+relu": ((0, ""), {"input": [(0, 128, 1), (0, 102, 128), (0, 82, 13056), (0, 5, 1070592)], "filter": [(0, 128, 1), (0, 3, 128), (0, 3, 384), (0, 128, 1152)], "bias": [(0, 128, 1)], "relu": [(0, 128, 1), (0, 100, 128), (0, 80, 12800), (0, 5, 1024000)]}),
    },
    "halide_b200_local_laplacian_sharded": {
        "input": ((0, ""), {"input": [(0, 10, 1), (0, 8, 10), (0, 3, 80)]}),
        "output": ((0, ""), {"output": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
        "input+output": ((0, ""), {"input": [(0, 0, 1), (0, 0, 0), (0, 0, 0)], "output": [(0, 0, 1), (0, 0, 0), (0, 0, 0)]}),
    },
}
