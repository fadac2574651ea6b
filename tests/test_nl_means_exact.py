"""On the CPU, for every case the bit-exact GPU tests of nl_means run (nl_means_exact.CASES): the content makes the kernel
mistakes worth catching visible, and the oracle agrees with an independent float64 restatement."""
import math

import numpy as np
import pytest

import nl_means_exact as E


@pytest.mark.parametrize("c", [c for c in E.CASES if c.need is not None], ids=lambda c: c.id)
def test_mutations_move_the_output(oracle, c):
    """Each probe offset left out, its neighbour read one column over, and the patch window one row down, each move the
    float64 result by at least c.need and by at least twice the oracle's distance from float64 on the same frame, so
    none of them can produce the oracle's bits."""
    inp, kw = E.frame(c)
    dev = E.rel(oracle.nl_means(inp, c.patch, c.search, c.sigma, **kw), E.nl_means64(inp, c.patch, c.search, c.sigma, **kw))
    need = max(c.need, 2 * dev)
    effects = E.mutation_effects(inp, c.patch, c.search, c.sigma, **kw)
    assert len(effects) == 2 * len(E.probe_offsets(c.search)) + 1
    if abs(c.sigma) >= 1e4:  # every weight is 1 (to float64's precision): the patch window cannot matter
        assert effects.pop("patch_row") < 1e-8
    weak = {k: v for k, v in effects.items() if not v >= need}
    assert not weak, f"mutations below {need}: {weak}"


def test_every_case_has_a_need_or_a_reason():
    for c in E.CASES:
        assert (c.need is None) == bool(c.why), c.id


@pytest.mark.parametrize("c", [c for c in E.CASES if abs(c.sigma) > 1e-10], ids=lambda c: c.id)
def test_oracle_within_float64_bound(oracle, c):
    """The oracle against nl_means64 on every case (at sigma 1e-20 the oracle's weights are NaN by design: see
    test_oracle_nan_weights_give_one)."""
    inp, kw = E.frame(c)
    got = oracle.nl_means(inp, c.patch, c.search, c.sigma, **kw)
    assert E.rel(got, E.nl_means64(inp, c.patch, c.search, c.sigma, **kw)) <= E.oracle_bound(c.search)


def test_oracle_nan_weights_give_one(oracle):
    """sigma 1e-20: sigma^2 * 9 is a denormal, -1 / it overflows to -inf, the centre weight is fast_exp(0 * -inf) = NaN
    and every other one fast_exp(-inf) = NaN (-inf - -inf in its range reduction).  The sums are NaN, and the final
    clamp(NaN, 0, 1) is 1.0: Halide's min and max select on a comparison, which is false for NaN."""
    (c,) = [c for c in E.group("sigma") if c.sigma == 1e-20]
    inp, kw = E.frame(c)
    f = np.float32
    assert math.isinf(f(-1) / (f(c.sigma) * f(c.sigma) * f(9)))
    assert (oracle.nl_means(inp, c.patch, c.search, c.sigma, **kw) == 1.0).all()


def test_outside_content_reaches_the_clamp(oracle):
    """The clamp cases: inputs span [-0.5, 1.5] and the unclamped result leaves [0, 1] on both sides."""
    for c in E.group("clamp"):
        inp, kw = E.frame(c)
        assert inp.min() < -0.4 and inp.max() > 1.4
        w, nb, _ = E.nl_means_terms(inp, c.patch, c.search, c.sigma, **kw)
        raw = sum(a * b for a, b in zip(w, nb)) / sum(w)
        assert (raw < 0).mean() > 0.05 and (raw > 1).mean() > 0.05
