"""The compiled-in weights of the integer-ratio kernels (smelter_b200/csrc/int_weights.h) against the oracle's weight
code, bit for bit, and the header against its generator (tools/gen_int_weights.py)."""
import os
import re

import numpy as np
import pytest

from oracle import oracle as orc

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "smelter_b200", "csrc", "int_weights.h")


def header_tables():
    """{S: (weights, inv)} as the header spells them, float32"""
    text = open(HEADER).read()
    res = {}
    for S, body in re.findall(r"int_weight<(\d)>\(int t\) \{\s*constexpr float w\[\d+\] = \{([^}]*)\}", text):
        w = np.array([float.fromhex(x.strip().rstrip("f")) for x in body.split(",") if x.strip()], np.float32)
        inv = re.search(r"int_inv<%s>\(\) \{ return ([^;]+);" % S, text).group(1).rstrip("f")
        res[int(S)] = (w, np.float32(float.fromhex(inv)))
    return res


@pytest.mark.parametrize("S", [2, 3, 4])
def test_header_weights_are_the_oracle_weights(S):
    """every tap and 1 / weight_sum of the S:1 mapping, at several output coordinates (the table is the same for all)"""
    w, inv = header_tables()[S]
    assert len(w) == 6 * S + 1
    first0 = orc.resample_weights(float(S), 0.0, 0)[0]
    for o in (0, 1, 7, 959, 3839):
        first, ow, ws = orc.resample_weights(float(S), 0.0, o)
        assert first == first0 + S * o   # the first tap moves with o, the weights do not
        assert np.array_equal(w.view(np.uint32), ow.astype(np.float32).view(np.uint32)), (S, o)
        assert (np.float32(1.0) / np.float32(ws)).view(np.uint32) == inv.view(np.uint32), (S, o)


def test_header_matches_generator():
    """the committed header is what tools/gen_int_weights.py writes"""
    import importlib.util
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "gen_int_weights.py")
    spec = importlib.util.spec_from_file_location("gen_int_weights", path)
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    assert open(HEADER).read() == gen.render()
