"""The zero tap of the integer-ratio weight rows (smelter_b200/csrc/int_weights.h): k_resample_tma3 issues no FFMA for the
trailing weights that are exactly zero (Cfg<S>::TAPS_NZ in resample_tma3.cuh, pinned there by a static_assert to 6 S).
That is only an identity if those weights are +0.0 bit for bit and no other weight of the row is skipped."""
import numpy as np
import pytest

from tests.test_int_weights import header_tables


def taps_nz(w):
    """the constexpr loop of Cfg<S>::taps_nz: taps in front of the trailing run of exact zeros"""
    n = len(w)
    while n > 0 and w[n - 1] == 0.0:
        n -= 1
    return n


@pytest.mark.parametrize("S", [2, 4])
def test_trailing_zero_tap_is_positive_zero_and_the_only_one(S):
    w, _ = header_tables()[S]
    assert len(w) == 6 * S + 1
    assert taps_nz(w) == 6 * S
    assert w[6 * S:].view(np.uint32).tolist() == [0]          # +0.0f, not -0.0f and not a denormal
    assert np.all(w[:6 * S] != 0.0)
    # no product of a decoded pixel (>= 1 / (255 * 12.92) unless 0) or an f16 ring value (>= 2^-24 unless 0) with a kept
    # weight is anywhere near the float32 underflow threshold, so an accumulator never reaches -0 by rounding
    assert np.min(np.abs(w[:6 * S])) >= 2.0 ** -10


def test_ratio_three_row_keeps_its_interior_near_zero_weights():
    """k_resample_fused_int<3> reads the same header and still issues every tap: its zeros sit at both ends, and the tiny
    interior weights are not zero"""
    w, _ = header_tables()[3]
    assert w[0] == 0.0 and w[18] == 0.0 and np.all(w[1:18] != 0.0)


def test_generator_ends_the_kept_rows_in_positive_zero():
    """what tools/gen_int_weights.py computes, before it is spelled as a literal"""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "gen_int_weights.py")
    spec = importlib.util.spec_from_file_location("gen_int_weights_zero_tap", path)
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    for S in (2, 4):
        gw, _ = gen.weights(S)
        assert gw[-1].view(np.uint32) == 0 and taps_nz(gw) == 6 * S
        assert gen.literal(gw[-1]) == "0x0p+0f"
