"""The device copy of the float pipelines' scalar primitives (halide_b200/csrc/hl_math.cuh), evaluated one primitive at a
time by halide_b200_selftest_math, against the CPU oracle's copy (oracle/halide_math.h, oracle_math_vec) bit for bit, and
against float64 for accuracy.

One-operand primitives are checked on all 2^32 float32 bit patterns, generated on the device in chunks.  An input is in
the *defined* domain when every float -> int conversion it causes is of a finite value inside int32 and k + 127 cannot
overflow; there the two copies must agree bit for bit (NaN results count as one value: their payload is not part of
Halide's semantics).  Inputs outside it are classified, and the mismatches found there are pinned per class.  Both
copies convert floor(x / ln 2) with one explicit, saturating conversion (NaN -> 0, clamped to [-256, 256], as cvt.rzi
followed by a clamp), so the exp and pow rows of that table are empty.
"""
import ctypes
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CHUNK = 1 << 24                # floats per device chunk: 64 MiB per float32 array, 128 MiB per float64 one
PEAK_LIMIT = 2 << 30           # device memory the module may hold at once (the machines are shared)
INV_LN2 = np.uint32(0x3FB8AA3B).view(np.float32)  # hl::kInvLn2, the 1/logf(2) both copies multiply by
TWO31 = 2.0 ** 31
DEVICE_ONLY = {"to_f32_u8": 10, "from_f32_u8": 11, "frame_val_u8": 12, "frame_narrow_u8": 13, "pair_u16_u8": 14}

# Mismatches between the two copies outside the defined domain, per primitive and class of input.  Before both copies
# converted floor(x / ln 2) through exp_k, x86 turned an out-of-range or NaN value into INT_MIN and the device saturated
# it (NaN -> 0): halide_exp differed on all 16777214 NaNs (x86 0, device NaN) and on all 818843113 x >= 2^31 ln 2, +inf
# included (x86 0, device +inf), and halide_pow likewise wherever log|x| * y was NaN or that large (x86 0, device NaN or
# +inf); fast_exp and k < -2^31 (0 on both) agreed.  What remains is clampf's: the device's fminf / fmaxf and the oracle's
# selects (min.f32 / max.f32 against compare-and-select, as Halide's GPU and x86 back-ends lower float min / max) differ
# where a bound is NaN and where two compared zeros differ in sign.
EXPECTED_MISMATCHES = {("clampf", "nan bound"): 24658, ("clampf", "signed zero tie"): 18}

# Worst error in float32 ulps against float64, over the inputs whose exact result is a normal float.  Inside Halide's
# test/correctness/vector_math.cpp ranges (x in [-4.5, 27.46875] for exp / fast_exp, (0, 27.46875] for log, and for pow
# x in [0.03125, 27.46875], y in [-0.28125, 1.716796875]) that test's thresholds apply; outside them the measured worst case
# is pinned (H100, measured on every float32 input of the one-operand primitives).
VM_LIMIT = {"halide_exp": 32, "halide_log": 8, "fast_exp": 64, "halide_pow": 64}
VM_RANGE = {"halide_exp": (-4.5, 27.46875), "fast_exp": (-4.5, 27.46875), "halide_log": (0.03125, 27.46875)}
# halide_log and halide_pow take no account of subnormal inputs (as in Halide): log(2^-149) is off by ~2e6 ulps
OUTSIDE_WORST = {"halide_exp": 2.200917797163129, "fast_exp": 81.21146368794143, "halide_log": 1998747.9003026187,
                 "halide_pow": 100529730.73504183}


def _bits(t):
    import torch
    return t.view(torch.int32)


def differ(g, o):
    """Elements where the device result g and the oracle result o differ as bit patterns (NaN == NaN)."""
    import torch
    return (_bits(g) != _bits(o)) & ~(torch.isnan(g) & torch.isnan(o))


def exp_classes(arg):
    """The classes of undefined input of an exp whose argument is `arg` (float32 tensor): the conversion of
    floor(arg / ln 2) is of a NaN, of a value >= 2^31 or of one < -2^31 (k + 127 then overflows, or the conversion is out
    of range).  Floats in [2^31 - 128, 2^31) do not exist, so k + 127 never overflows for an in-range k."""
    import torch
    k = torch.floor(arg * float(INV_LN2))
    return {"nan": torch.isnan(k), "k >= 2^31": k >= TWO31, "k < -2^31": k < -TWO31}


class Tally:
    def __init__(self):
        self.mismatch, self.domain, self.samples = {}, {}, {}

    def add(self, name, bad, classes, inputs, g, o):
        import torch
        undefined = torch.zeros_like(bad)
        for cls, m in classes.items():
            undefined |= m
            n = int(m.sum())
            if n:
                self.domain[(name, cls)] = self.domain.get((name, cls), 0) + n
            nb = int((bad & m).sum())
            if nb:
                self.mismatch[(name, cls)] = self.mismatch.get((name, cls), 0) + nb
                if (name, cls) not in self.samples:
                    i = int(torch.nonzero(bad & m)[0])
                    self.samples[(name, cls)] = tuple(float(t[i]) for t in (*inputs, g, o))
        defined_bad = bad & ~undefined
        if bool(defined_bad.any()):
            i = int(torch.nonzero(defined_bad)[0])
            vals = [float(t[i]) for t in inputs]
            pytest.fail(f"{name}{tuple(vals)}: device {float(g[i])!r} ({int(_bits(g)[i]) & 0xffffffff:#010x}), oracle "
                        f"{float(o[i])!r} ({int(_bits(o)[i]) & 0xffffffff:#010x}) in the defined domain "
                        f"({int(defined_bad.sum())} such inputs in this chunk)")

    def check(self, names):
        got = {k: v for k, v in self.mismatch.items() if k[0] in names}
        for k, v in sorted(self.samples.items()):
            if k[0] in names:
                print(f"undefined-domain mismatch {k}: {got[k]} inputs (of {self.domain[k]}), e.g. inputs/device/oracle {v}")
        want = {k: v for k, v in EXPECTED_MISMATCHES.items() if k[0] in names}
        assert got == want


@pytest.fixture(scope="module")
def dev(hb):
    """run(fn, a, b=None, dtype): the device hook on torch tensors; checks the module's peak device memory at the end."""
    import torch
    l = hb.load_library()
    l.halide_b200_selftest_math.restype = ctypes.c_int
    l.halide_b200_selftest_math.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong]
    from oracle import pyoracle
    codes = dict(pyoracle.MATH_FN, **DEVICE_ONLY)

    def run(fn, a, b=None, dtype=torch.float32):
        out = torch.empty(a.shape, dtype=dtype, device=a.device)
        r = l.halide_b200_selftest_math(codes[fn], a.data_ptr(), None if b is None else b.data_ptr(), out.data_ptr(), a.numel())
        assert r == 0, f"halide_b200_selftest_math({fn}) returned {r}"
        return out

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield run
    peak = torch.cuda.max_memory_allocated()
    print(f"\ntest_hl_math_gpu: peak device memory {peak / 2 ** 20:.0f} MiB, {time.perf_counter() - t0:.1f} s")
    assert peak <= PEAK_LIMIT


@pytest.fixture(scope="module")
def tally():
    return Tally()


@pytest.fixture(scope="module")
def host_buf():
    import torch
    return torch.empty(CHUNK, dtype=torch.float32, pin_memory=True)


def oracle_on(oracle, host_buf, fn, a, b=None):
    """The oracle's `fn` on device tensor a (and b), computed on the host and brought back to the device."""
    import torch
    a1 = a.reshape(-1)
    b1 = None if b is None else b.reshape(a1.numel(), -1)
    res = torch.empty_like(a1)
    for s in range(0, a1.numel(), CHUNK):
        n = min(CHUNK, a1.numel() - s)
        out = host_buf[:n]
        oracle.math_vec(fn, a1[s:s + n].cpu().numpy(), None if b1 is None else b1[s:s + n].cpu().numpy(), out=out.numpy())
        res[s:s + n].copy_(out, non_blocking=True)
        torch.cuda.synchronize()
    return res.reshape(a.shape)


def all_float_chunks(lo=-(1 << 31), hi=1 << 31):
    """Every float32 bit pattern in [lo, hi) (as int32), in device chunks."""
    import torch
    for s in range(lo, hi, CHUNK):
        yield torch.arange(s, min(s + CHUNK, hi), dtype=torch.int64, device="cuda").to(torch.int32).view(torch.float32)


def ulp_err(got, ref):
    """|got - ref| in float32 ulps of ref (float64), for ref whose magnitude is a normal float32."""
    import torch
    _, e = torch.frexp(ref)
    return (got.double() - ref).abs() / torch.ldexp(torch.ones_like(ref), (e - 24))


def normal_f32(ref):
    a = ref.abs()
    return (a >= 2.0 ** -126) & (a <= float(np.finfo(np.float32).max))


class Worst:
    def __init__(self):
        self.v = {}

    def add(self, key, err, args):
        import torch
        if err.numel() == 0:
            return
        i = int(torch.argmax(err))
        e = float(err[i])
        if e > self.v.get(key, (-1.0,))[0]:
            self.v[key] = (e, tuple(float(a[i]) for a in args))


@pytest.fixture(scope="module")
def worst():
    return Worst()


# ---- one operand, every float32 ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fn", ["halide_exp", "fast_exp", "halide_log", "clamp01"])
def test_one_operand_every_float_matches_oracle(dev, oracle, host_buf, tally, worst, fn):
    import torch
    for x in all_float_chunks():
        g = dev(fn, x)
        o = oracle_on(oracle, host_buf, fn, x)
        classes = exp_classes(x) if fn in ("halide_exp", "fast_exp") else {}
        tally.add(fn, differ(g, o), classes, (x,), g, o)
        if fn == "clamp01":
            continue
        ref = torch.log(x.double()) if fn == "halide_log" else torch.exp(x.double())
        ok = normal_f32(ref)
        lo, hi = VM_RANGE[fn]
        inside = ok & (x >= lo) & (x <= hi)
        err = ulp_err(g[ok], ref[ok])
        worst.add((fn, "inside"), ulp_err(g[inside], ref[inside]), (x[inside],))
        worst.add((fn, "outside"), err[~inside[ok]], (x[ok][~inside[ok]],))
        del ref, ok, inside, err
    if fn != "clamp01":
        for where in ("inside", "outside"):
            print(f"{fn} worst ulps {where} vector_math's range: {worst.v.get((fn, where))}")
    tally.check({fn})
    if fn != "clamp01":
        assert worst.v[(fn, "inside")][0] <= VM_LIMIT[fn]
        if fn in OUTSIDE_WORST:
            assert worst.v[(fn, "outside")][0] == pytest.approx(OUTSIDE_WORST[fn], abs=1e-3)


def test_clamp01_is_halide_clamp(dev):
    """clamp(v, 0, 1) as Halide's select-based min / max: NaN -> 1, -0 -> +0 (the oracle comparison covers every other
    input)."""
    import torch
    x = torch.tensor([float("nan"), -0.0, -float("inf"), float("inf"), 0.5, 1.0000001], device="cuda")
    got = dev("clamp01", x).cpu().numpy()
    assert got.view(np.uint32).tolist() == np.array([1.0, 0.0, 0.0, 1.0, 0.5, 1.0], np.float32).view(np.uint32).tolist()


# ---- halide_pow --------------------------------------------------------------------------------------------------------
def _pow_check(dev, oracle, host_buf, tally, x, y, what):
    g = dev("halide_pow", x, y)
    o = oracle_on(oracle, host_buf, "halide_pow", x, y)
    arg = dev("halide_log", x.abs()) * y
    tally.add("halide_pow", differ(g, o), exp_classes(arg), (x, y), g, o)
    return g


def _rand_floats(gen, n, exp_lo, exp_hi, signed=True):
    import torch
    e = torch.randint(exp_lo, exp_hi + 1, (n,), generator=gen, device="cuda", dtype=torch.int32)
    m = torch.randint(0, 1 << 23, (n,), generator=gen, device="cuda", dtype=torch.int32)
    s = torch.randint(0, 2, (n,), generator=gen, device="cuda", dtype=torch.int32) if signed else torch.zeros_like(e)
    return ((s << 31) | (e << 23) | m).view(torch.float32)


def test_pow_every_exponent_pair(dev, oracle, host_buf, tally, worst):
    """Every (biased exponent of x, biased exponent of y) pair, zeros / subnormals / inf / NaN included, 64 random
    mantissas and signs each."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(7)
    ex, ey = torch.meshgrid(torch.arange(256, device="cuda", dtype=torch.int32),
                            torch.arange(256, device="cuda", dtype=torch.int32), indexing="ij")
    ex, ey = ex.reshape(-1).repeat(64), ey.reshape(-1).repeat(64)

    def with_exp(e):
        m = torch.randint(0, 1 << 23, e.shape, generator=gen, device="cuda", dtype=torch.int32)
        s = torch.randint(0, 2, e.shape, generator=gen, device="cuda", dtype=torch.int32)
        return ((s << 31) | (e << 23) | m).view(torch.float32)

    x, y = with_exp(ex), with_exp(ey)
    g = _pow_check(dev, oracle, host_buf, tally, x, y, "exponent pairs")
    ref = torch.pow(x.double().abs(), y.double())
    ok = normal_f32(ref) & (x > 0)
    worst.add(("halide_pow", "outside"), ulp_err(g[ok], ref[ok]), (x[ok], y[ok]))


def test_pow_unit_interval_every_float(dev, oracle, host_buf, tally):
    """camera_pipe's use: every float in [0, 1] raised to 1 / gamma for the harness's gamma and the extremes its tests
    take."""
    import torch
    for gamma in (2.0, 0.25, 10.0, 1.0 / 2.2):
        y = float(np.float32(1.0) / np.float32(gamma))
        for x in all_float_chunks(0, 0x3F800001):
            _pow_check(dev, oracle, host_buf, tally, x, torch.full_like(x, y), f"gamma {gamma}")


def test_pow_dense_y_grid(dev, oracle, host_buf, tally):
    """Every 4096th float in [0, 1] and the curve's own x / 1023 against 4096 exponents from -64 to 64."""
    import torch
    xs = torch.cat([torch.arange(0, 0x3F800001, 4096, dtype=torch.int32, device="cuda").view(torch.float32),
                    torch.arange(1024, device="cuda", dtype=torch.float32) / 1023.0])
    ys = torch.linspace(-64, 64, 4096, device="cuda", dtype=torch.float32)
    for i in range(0, ys.numel(), 32):
        yy = ys[i:i + 32]
        x, y = torch.meshgrid(xs, yy, indexing="ij")
        _pow_check(dev, oracle, host_buf, tally, x.reshape(-1).contiguous(), y.reshape(-1).contiguous(), "dense y")


SPECIALS = [0.0, -0.0, float("inf"), -float("inf"), float("nan"), 1.0, -1.0, 2.0, -2.0, 0.5, -0.5, 3.0, -3.0, 2.5, -2.5,
            1e-45, -1e-45, 1e-38, 3.4028235e38, -3.4028235e38, 1e10, -1e10, 127.0, 128.0, -126.0, -149.0, -150.0, 2.0 ** 24,
            2.0 ** 24 + 2, -(2.0 ** 24 + 2), 1.0000001, 0.99999994]


def test_pow_specials(dev, oracle, host_buf, tally):
    """Zeros, infinities, NaN, negative x with integer and non-integer y, every pair."""
    import torch
    s = torch.tensor(SPECIALS, dtype=torch.float32, device="cuda")
    x, y = torch.meshgrid(s, s, indexing="ij")
    x, y = x.reshape(-1).contiguous(), y.reshape(-1).contiguous()
    g = _pow_check(dev, oracle, host_buf, tally, x, y, "specials").cpu()
    xc, yc = x.cpu(), y.cpu()
    # Halide's pow: 1 for y = 0 whatever x (NaN included), 0 for x = 0 and y != 0, NaN for x < 0 and non-integer y
    for i in range(x.numel()):
        xi, yi, gi = float(xc[i]), float(yc[i]), float(g[i])
        if yi == 0 and not xi > 0:
            assert gi == 1.0, (xi, yi, gi)
        elif xi == 0:
            assert gi == 0.0, (xi, yi, gi)
        elif xi < 0 and np.isfinite(yi) and yi != np.floor(yi):
            assert np.isnan(gi), (xi, yi, gi)


def test_pow_vector_math_range(dev, oracle, host_buf, tally, worst):
    """vector_math.cpp's pow inputs (a = (i / 16 - 9) / 2 > 0, y = (j / 16 - 9) / 32 for i, j in 0 .. 1023) and 2^24 random
    pairs from the same box: within 64 ulps of float64, and bit for bit against the oracle."""
    import torch
    v = (torch.arange(1024, device="cuda", dtype=torch.float32) * 0.0625 - 9.0) * 0.5
    x, y = torch.meshgrid(v[v > 0], v / 16.0, indexing="ij")
    gen = torch.Generator(device="cuda").manual_seed(11)
    xr = torch.rand(1 << 24, generator=gen, device="cuda") * (27.46875 - 0.03125) + 0.03125
    yr = torch.rand(1 << 24, generator=gen, device="cuda") * (1.716796875 + 0.28125) - 0.28125
    x = torch.cat([x.reshape(-1), xr[xr > 0]])
    y = torch.cat([y.reshape(-1), yr[xr > 0]])
    g = _pow_check(dev, oracle, host_buf, tally, x, y, "vector_math range")
    ref = torch.pow(x.double(), y.double())
    ok = normal_f32(ref)
    worst.add(("halide_pow", "inside"), ulp_err(g[ok], ref[ok]), (x[ok], y[ok]))
    print(f"halide_pow worst ulps inside vector_math's range: {worst.v.get(('halide_pow', 'inside'))}, outside (exponent "
          f"pairs): {worst.v.get(('halide_pow', 'outside'))}")
    tally.check({"halide_pow"})
    assert worst.v[("halide_pow", "inside")][0] <= VM_LIMIT["halide_pow"]
    if "halide_pow" in OUTSIDE_WORST:
        assert worst.v[("halide_pow", "outside")][0] == pytest.approx(OUTSIDE_WORST["halide_pow"], abs=1e-3)


# ---- clampf, lerpf, evaluate_polynomial -------------------------------------------------------------------------------
def _operands(seed, n=1 << 22):
    """Random bit patterns (every class of float) and values from [-2, 2], interleaved with every triple of specials."""
    import torch
    gen = torch.Generator(device="cuda").manual_seed(seed)
    raw = torch.randint(-(1 << 31), 1 << 31, (n, 3), generator=gen, device="cuda", dtype=torch.int64).to(torch.int32)
    small = torch.rand((n, 3), generator=gen, device="cuda") * 4 - 2
    s = torch.tensor(SPECIALS[:12], dtype=torch.float32, device="cuda")
    sp = torch.cartesian_prod(s, s, s)
    return torch.cat([raw.view(torch.float32), small, sp]).contiguous()


def test_clampf_matches_oracle(dev, oracle, host_buf, tally):
    """clampf(a, lo, hi) = max(min(a, hi), lo).  The device's fminf / fmaxf and the oracle's selects differ, as Halide
    lets min / max of floats differ across targets, where a bound is NaN and where two compared zeros differ in sign;
    those inputs form the undefined classes."""
    import torch
    t = _operands(3)
    a, b = t[:, 0].contiguous(), t[:, 1:].contiguous()
    lo, hi = b[:, 0], b[:, 1]
    g = dev("clampf", a, b)
    o = oracle_on(oracle, host_buf, "clampf", a, b)
    m = torch.where(a < hi, a, hi)
    zero_tie = ((m == 0) & (hi == 0) & (torch.signbit(a) != torch.signbit(hi)) & (a == 0)) | \
               ((m == 0) & (lo == 0) & (torch.signbit(m) != torch.signbit(lo)))
    classes = {"nan bound": torch.isnan(lo) | torch.isnan(hi), "signed zero tie": zero_tie}
    tally.add("clampf", differ(g, o), classes, (a, lo, hi), g, o)
    tally.check({"clampf"})


@pytest.mark.parametrize("fn", ["lerpf", "poly8", "poly10", "poly7"])
def test_float_expressions_match_oracle(dev, oracle, host_buf, tally, fn):
    """lerpf(zero, one, w) and evaluate_polynomial with even and odd coefficient counts and zero coefficients: plain IEEE
    expressions, defined everywhere."""
    t = _operands(5)
    a = t[:, 0].contiguous()
    b = t[:, 1:].contiguous() if fn == "lerpf" else None
    g = dev(fn, a, b)
    o = oracle_on(oracle, host_buf, fn, a, b)
    tally.add(fn, differ(g, o), {}, (a,), g, o)


# ---- 8-bit conversions, exhaustively ----------------------------------------------------------------------------------
def test_u8_to_f32_every_code(dev):
    import torch
    from halide_b200 import image_io
    codes = np.arange(256, dtype=np.uint8)
    got = dev("to_f32_u8", torch.from_numpy(codes).cuda()).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), image_io.convert(codes, np.float32).view(np.uint32))


def test_f32_to_u8_every_float_in_unit_interval(dev):
    """Every float in [0, 1], and its neighbours outside: -0, the negative subnormals near it and the 2^16 floats above 1."""
    import torch
    from halide_b200 import image_io
    above = np.arange(0x3F800001, 0x3F800001 + (1 << 16), dtype=np.int32)
    below = np.concatenate([np.array([-(1 << 31)], np.int64), -(1 << 31) + np.arange(1, 1 << 16, dtype=np.int64)]).astype(np.int32)
    for s in list(range(0, 0x3F800001, CHUNK)) + ["edges"]:
        if s == "edges":
            xi = torch.from_numpy(np.concatenate([above, below])).cuda()
        else:
            xi = torch.arange(s, min(s + CHUNK, 0x3F800001), dtype=torch.int32, device="cuda")
        x = xi.view(torch.float32)
        got = dev("from_f32_u8", x, dtype=torch.uint8).cpu().numpy()
        want = image_io.convert(x.cpu().numpy(), np.uint8)
        if not np.array_equal(got, want):
            i = int(np.flatnonzero(got != want)[0])
            pytest.fail(f"frame_from_f32<uint8_t>({float(x[i])!r}) = {got[i]}, convert gives {want[i]}")


def test_local_laplacian_u8_u16_pair_every_code(dev):
    """frame_val (u8 -> u16 as float) on all 256 codes, pair_u16 on all 65536 byte pairs and frame_narrow (u16 -> u8) on
    all 65536 codes, against the reference's conversions."""
    import torch
    from halide_b200 import image_io
    codes = np.arange(256, dtype=np.uint8)
    wide = dev("frame_val_u8", torch.from_numpy(codes).cuda()).cpu().numpy()
    assert np.array_equal(wide, image_io.convert(codes, np.uint16).astype(np.float32))
    words = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    pair = dev("pair_u16_u8", torch.from_numpy(words.view(np.int16)).cuda(), dtype=torch.int32).cpu().numpy().view(np.uint32)
    lo = image_io.convert((words & 0xFF).astype(np.uint8), np.uint16).astype(np.uint32)
    hi = image_io.convert((words >> 8).astype(np.uint8), np.uint16).astype(np.uint32)
    assert np.array_equal(pair, lo | (hi << 16))
    narrow = dev("frame_narrow_u8", torch.from_numpy(words.view(np.int16)).cuda(), dtype=torch.uint8).cpu().numpy()
    assert np.array_equal(narrow, image_io.convert(words, np.uint8))


# ---- camera_pipe's tables -----------------------------------------------------------------------------------------------
CP_LEVELS = [(25, 1023), (0, 1023), (0, 1), (1022, 1023), (-100, 1023), (500, 500), (600, 400), (25, 4000), (0, 1 << 30)]

# The scalar bounds at which camera_pipe's halide_pow calls leave the defined domain (floor(arg / ln 2) of a NaN, or out
# of int32), derived below from the float32 expressions the curve evaluates.  contrast: 2^(contrast / 100) is defined
# for contrast in [CONTRAST_LO, CONTRAST_HI] and not for NaN.  gamma (black 25, white 1023, where the smallest curve
# input above black is 1 / 998): x^(1 / gamma) is defined for every used x when gamma >= GAMMA_POS or gamma <= GAMMA_NEG,
# including +-inf, and not for gamma in (GAMMA_NEG, GAMMA_POS), 0 included, nor for NaN.
CP_BOUNDS = {"contrast_lo": -214748381184.0, "contrast_hi": 214748348416.0, "gamma_pos": 4.639334694189756e-09,
             "gamma_neg": -4.639335138278966e-09}


def _cp_tables(hb, m32, m70, scalars, levels):
    import torch
    l = hb.load_library()
    n = len(scalars)
    sc = np.ascontiguousarray(scalars, np.float32)
    lv = np.ascontiguousarray(levels, np.int32)
    matrix = torch.empty((n, 12), dtype=torch.int16, device="cuda")
    curve = torch.empty((n, 1024), dtype=torch.uint8, device="cuda")
    s32 = torch.empty(n, dtype=torch.uint8, device="cuda")
    f = ctypes.c_void_p
    r = l.halide_b200_camera_pipe_tables(f(m32.data_ptr()), f(m70.data_ptr()), sc.ctypes.data_as(f), lv.ctypes.data_as(f),
                                         ctypes.c_int(n), f(matrix.data_ptr()), f(curve.data_ptr()), f(s32.data_ptr()))
    assert r == 0
    return matrix.cpu().numpy(), curve.cpu().numpy(), s32.cpu().numpy()


def _float_between(pred, lo, hi):
    """The float32 f in (lo, hi] at which the monotone predicate turns from False (at lo) to True (at hi): bisection on
    the float ordering (same-sign floats order like their bit patterns)."""
    a, b = int(np.float32(lo).view(np.int32)), int(np.float32(hi).view(np.int32))
    as_f = lambda i: float(np.int32(i).view(np.float32))  # noqa: E731
    assert not pred(as_f(a)) and pred(as_f(b))
    while abs(b - a) > 1:
        m = (a + b) // 2
        if pred(as_f(m)):
            b = m
        else:
            a = m
    return as_f(b)


def _exp_arg_defined(arg):
    with np.errstate(all="ignore"):
        k = np.floor(np.asarray(arg, np.float32) * INV_LN2)
    return bool(np.all(np.isfinite(k) & (k >= -TWO31) & (k < TWO31)))


def test_camera_pipe_curve_scalar_bounds(oracle):
    """Derive where camera_pipe's halide_pow arguments leave the defined domain, from the float32 expressions the tables
    evaluate (contrast * 0.01f, halide_log(2) or halide_log(x) times 1 / gamma, times 1 / ln 2, floored)."""
    l2 = np.float32(oracle.math_vec("halide_log", np.array([2.0], np.float32))[0])
    contrast_ok = lambda c: _exp_arg_defined(l2 * (np.float32(c) * np.float32(0.01)))  # noqa: E731
    c_hi = _float_between(lambda c: not contrast_ok(c), 0.0, 1e30)
    c_hi = float(np.nextafter(np.float32(c_hi), np.float32(0)))
    c_lo = _float_between(lambda c: not contrast_ok(c), -0.0, -1e30)
    c_lo = float(np.nextafter(np.float32(c_lo), np.float32(0)))
    x = np.arange(1024, dtype=np.float32)
    xf = np.clip((x[26:] - np.float32(25)) * (np.float32(1) / np.float32(998)), 0, 1).astype(np.float32)
    lx = oracle.math_vec("halide_log", xf)
    def gamma_ok(g):
        with np.errstate(all="ignore"):
            return _exp_arg_defined(lx * (np.float32(1) / np.float32(g)))
    g_pos = _float_between(gamma_ok, 0.0, 1.0)
    g_neg = _float_between(gamma_ok, -0.0, -1.0)
    got = {"contrast_lo": c_lo, "contrast_hi": c_hi, "gamma_pos": g_pos, "gamma_neg": g_neg}
    print(f"camera_pipe scalar bounds: {got}")
    assert contrast_ok(c_hi) and not contrast_ok(np.nextafter(np.float32(c_hi), np.float32(np.inf)))
    assert contrast_ok(c_lo) and not contrast_ok(np.nextafter(np.float32(c_lo), np.float32(-np.inf)))
    assert not contrast_ok(np.nan) and gamma_ok(np.inf) and gamma_ok(-np.inf) and not gamma_ok(0.0) and not gamma_ok(np.nan)
    assert got == CP_BOUNDS


def _sweep():
    gammas = sorted(set([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 1e-9, 4e-9, 5e-9, 1e-8, -1e-9, -5e-9, -1e-8,
                         -1.0, -0.5, -2.2, 1e-3, 0.01, 0.1, 0.25, 0.5, 1 / 2.2, 1.0, 2.0, 2.2, 4.0, 10.0, 100.0, 1e6, 1e30]
                        + [float(g) for g in np.geomspace(0.05, 20, 24, dtype=np.float32)]), key=lambda v: (np.isnan(v), v))
    contrasts = [-float("inf"), -1e30, -2.2e11, -2.1e11, -1e4, -200.0, -100.0, -50.0, 0.0, 25.0, 50.0, 100.0, 150.0, 200.0,
                 1e3, 1e4, 12700.0, 12800.0, 2.1e11, 2.2e11, 1e30, float("inf"), float("nan")]
    return [(3700.0, g, c, 1.0) for g in gammas for c in contrasts]


def test_camera_pipe_tables_match_oracle_dense_sweep(hb, oracle):
    """The device tables against oracle_camera_pipe_tables on every (gamma, contrast, black / white) of the sweep,
    bit for bit, defined domain or not, and the matrix and sharpen strength at the colour temperatures and strengths the
    filter accepts."""
    import torch
    from util import CP_M3200, CP_M7000
    m32, m70 = (torch.from_numpy(np.ascontiguousarray(m)).cuda() for m in (CP_M3200, CP_M7000))
    scalars = _sweep()
    scalars += [(t, 2.0, 50.0, s) for t in (1000.0, 2000.0, 3200.0, 3700.0, 7000.0, 20000.0, 1e5)
                for s in (-1.0, 0.0, 0.03, 1 / 32, 1.0, 7.96875, 100.0, float("inf"), float("nan"))]
    rows = [(s, lv) for lv in CP_LEVELS for s in scalars]
    matrix, curve, s32 = _cp_tables(hb, m32, m70, [r[0] for r in rows], [r[1] for r in rows])
    for i, ((t, g, c, s), (b, w)) in enumerate(rows):
        wm, wc, ws = oracle.camera_pipe_tables(CP_M3200, CP_M7000, t, g, c, s, b, w)
        if not np.array_equal(curve[i], wc):
            j = int(np.flatnonzero(curve[i] != wc)[0])
            pytest.fail(f"curve at gamma {g}, contrast {c}, black {b}, white {w}: entry {j} device {curve[i][j]} oracle {wc[j]}")
        assert np.array_equal(matrix[i].reshape(3, 4), wm) and s32[i] == ws, (t, s)
    assert len(rows) >= 5000
