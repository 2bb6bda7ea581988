"""CPU tier: tools/conv_tc_fit.py recovers the per-step slope and the K-independent part of a tile from a per-shape table."""
import math
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import conv_tc_fit  # noqa: E402


def _row(kernel, ci, co, k, dil, L, slope_us, fixed_us, per_step, sms):
    r = dict(shape=f"rb c{co} k{k} d{dil}", Cin=ci, Cout=co, K=k, dil=dil, L=L, B=32, kernel=kernel, per_step=per_step)
    per_sm = conv_tc_fit.tiles(r) / sms
    r["ms"] = (slope_us * k * math.ceil(ci / 16) + fixed_us) * per_sm / 1e3
    return r


@pytest.mark.parametrize("kernel,ch,L", [("tct", 128, 61441), ("tc", 256, 10240)])
def test_fit_recovers_slope_and_fixed_part(kernel, ch, L):
    rows = [_row(kernel, ch, ch, k, 3, L, 0.2, 37.0, 2, 132) for k in (3, 7, 11)]
    rows.append(_row(kernel, ch, ch, 7, 1, L, 0.2, 50.0, 4, 132))   # a single K: no fit for that dilation
    (f,) = conv_tc_fit.fit(rows, 132, 1.5)
    assert (f["kernel"], f["dil"], f["K"]) == (kernel, 3, [3, 7, 11])
    assert f["slope_cycles"] == pytest.approx(0.2 * 1.5e3)
    assert f["fixed_us"] == pytest.approx(37.0)
    tiles_per_sm = conv_tc_fit.tiles(rows[0]) / 132
    assert f["fixed_ms_per_step"] == pytest.approx(3 * 2 * 37.0 * tiles_per_sm / 1e3)
