"""The rounding-bracket oracle (``tests/rounding.py``) on constructed values, without a GPU."""

from __future__ import annotations

import numpy as np
import pytest
import rounding as rd

H1 = 2.0 ** -10      # float16 ulp at 1
S1 = 2.0 ** -23      # float32 ulp at 1


def test_gamma_matches_its_definition():
    assert rd.gamma(0) == 0.0
    assert rd.gamma(1) == pytest.approx(2.0 ** -53, rel=1e-15)
    n = 1024
    assert rd.gamma(n) == pytest.approx(n * 2.0 ** -53 / (1 - n * 2.0 ** -53), rel=1e-15)
    assert np.all(np.diff(rd.gamma(np.arange(1, 100))) > 0)


def test_exact_midpoint_has_two_answers_only_with_a_bound():
    mid = 1.0 + H1 / 2                                        # between 1 and 1 + 2^-10: ties to even -> 1
    assert rd.check(np.float16(1.0), mid, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError, match="outside the rounding bracket"):
        rd.check(np.float16(1.0 + H1), mid, 0.0, rd.f16, what="host")
    # any b > 0 puts the boundary inside the interval: both neighbours become acceptable, counted as two-value
    assert rd.check(np.float16(1.0 + H1), mid, 1e-12, rd.f16, what="host") == 1
    assert rd.check(np.float16(1.0), mid, 1e-12, rd.f16, what="host") == 1
    mid3 = 1.0 + 3 * H1 / 2                                   # between 1 + 2^-10 (odd) and 1 + 2^-9: ties up
    assert rd.check(np.float16(1.0 + 2 * H1), mid3, 0.0, rd.f16, what="host") == 0
    m32 = 1.0 + S1 / 2
    assert rd.check(np.float32(1.0), m32, 0.0, rd.f32, what="host") == 0


def test_one_float64_ulp_either_side_of_a_midpoint():
    mid = 1.0 + H1 / 2
    below, above = np.nextafter(mid, 0.0), np.nextafter(mid, 2.0)
    assert rd.check(np.float16(1.0), below, 0.0, rd.f16, what="host") == 0
    assert rd.check(np.float16(1.0 + H1), above, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError):
        rd.check(np.float16(1.0), above, 0.0, rd.f16, what="host")
    # a bound of one float64 ulp reaches the midpoint from either side: both answers are acceptable
    ulp = np.spacing(mid)
    assert rd.check(np.float16(1.0), above, ulp, rd.f16, what="host") == 1
    assert rd.check(np.float16(1.0), below, ulp, rd.f16, what="host") == 0    # reaches the tie, which goes to even
    # two ulps above, a bound of one ulp stays clear of it
    assert rd.check(np.float16(1.0 + H1), above + ulp, ulp, rd.f16, what="host") == 0


def test_fp16_overflow_at_65520():
    assert rd.f16(65520.0) == np.inf and rd.f16(-65520.0) == -np.inf
    assert rd.f16(np.nextafter(65520.0, 0.0)) == 65504.0
    v = np.array([65520.0, -65520.0, 70000.0, 1e300, np.nextafter(65520.0, 0.0)])
    out = np.array([np.inf, -np.inf, np.inf, np.inf, 65504.0], np.float32)   # fp16 results widened to float32
    assert rd.check(out, v, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError):
        rd.check(np.array([65504.0], np.float32), [65520.0], 0.0, rd.f16, what="host")
    # a bound that straddles the overflow threshold: 65504 and inf are neighbours in float16
    assert rd.check(np.array([np.inf], np.float32), [65520.0], 1.0, rd.f16, what="host") == 1


def test_subnormal_halves():
    tiny = 2.0 ** -24                                         # smallest float16 subnormal
    assert rd.f16(tiny / 2) == 0.0                            # tie -> even (0)
    assert rd.f16(3 * tiny / 2) == 2 * tiny                   # tie -> even (2 tiny)
    assert rd.f16(np.nextafter(tiny / 2, 1.0)) == tiny
    v = np.array([tiny / 2, 3 * tiny / 2, np.nextafter(tiny / 2, 1.0), -tiny / 2, 5 * tiny / 4])
    out = np.array([0.0, 2 * tiny, tiny, -0.0, tiny], np.float32)
    assert rd.check(out, v, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError):
        rd.check(np.array([tiny], np.float32), [tiny / 2], 0.0, rd.f16, what="host")


def test_double_rounding_case_takes_the_direct_answer():
    v = 1.0 + H1 / 2 + 2.0 ** -40          # just past an fp16 midpoint; float32 rounds it onto the midpoint
    direct = rd.f16(v)
    via_f32 = np.float32(v).astype(np.float16)
    assert direct == 1.0 + H1 and via_f32 == 1.0
    assert rd.check(np.float32(direct), v, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError):
        rd.check(np.float32(via_f32), v, 0.0, rd.f16, what="host")


def test_chains_of_roundings_and_nan():
    def cos_chain(x):   # 1 - (1 - f32(s)) in float32 arithmetic
        one = np.float32(1.0)
        return one - (one - rd.f32(np.clip(x, -1.0, 1.0)))

    s = np.array([0.3, 0.999999, -0.7, 1.0 + 1e-12])
    assert rd.check(cos_chain(s), s, 1e-15, cos_chain, what="host") == 0
    assert cos_chain(0.1) != rd.f32(0.1) and cos_chain(-0.7) != rd.f32(-0.7)   # the round trip moves values below 0.5
    nan = np.array([np.nan, 1.0])
    assert rd.check(np.array([np.nan, 1.0], np.float16), nan, 0.0, rd.f16, what="host") == 0
    with pytest.raises(AssertionError):
        rd.check(np.array([0.0, 1.0], np.float16), nan, 0.0, rd.f16, what="host")


def test_loose_bound_is_refused():
    v = np.linspace(1.0, 2.0, 1000)
    with pytest.raises(AssertionError, match="two-value branch"):
        rd.check(rd.f16(v), v, 1e-2, rd.f16, what="host")
    with pytest.raises(AssertionError, match="two-value branch"):
        rd.check(rd.f16(v), v, 2.0 ** -12, rd.f16, what="host")


def test_bound_spanning_several_steps_accepts_the_interval_only():
    v = 1.0 + 2 * H1                              # b covers 1 .. 1 + 4 2^-10
    assert rd.check(np.float16(1.0 + H1), v, 2 * H1, rd.f16, what="host") == 1
    assert rd.check(np.float16(1.0 + 4 * H1), v, 2 * H1, rd.f16, what="host") == 1
    with pytest.raises(AssertionError, match="outside the rounding bracket"):
        rd.check(np.float16(1.0 + 5 * H1), v, 2 * H1, rd.f16, what="host")
