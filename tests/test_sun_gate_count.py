"""Host-side count of the (lane, step) pairs the PV sun gate loads (synthetic.lit_lane_steps),
against the float64 solar position of the oracle."""

import warnings

import numpy as np
import pytest

import atlite_oracle as O
from atlite_b200 import synthetic as syn


def _oracle_count(time, x, y, thr_deg, vec):
    d = {"time": time, "lon": x, "lat": y}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        alt = O.solar_position(d)["altitude"]  # (time, y, x) float64
    nt, ny, nx = alt.shape
    up = alt >= np.radians(thr_deg)
    if vec:
        up = up[:, :, np.minimum(np.arange(-(-nx // 4) * 4), nx - 1)].reshape(nt, ny, -1, 4).any(-1)
    else:
        up = up[:, np.minimum(np.arange(-(-ny // 4) * 4), ny - 1), :].reshape(nt, -1, 4, nx).any(2)
    return int(up.sum()), up.size


@pytest.mark.parametrize("vec", [True, False])
def test_lit_lane_steps_agree_with_the_oracle_altitude(vec):
    x, y = syn.make_coords(61, 43, -180.0, -88.0, 6.0, 4.2)  # global, neither dimension a multiple of 4
    time = syn.make_time(24 * 3 + 24 * 170)[24 * 170:]
    lit, total = syn.lit_lane_steps(time, x, y, vec=vec)
    want, n = _oracle_count(time, x, y, 1.0, vec)
    assert total == n
    assert 0.3 < lit / total < 0.8
    # float32 tables vs float64: only lanes whose brightest cell sits at the threshold may differ
    assert abs(lit - want) <= 2e-3 * total


def test_lit_lane_steps_limits():
    x, y = syn.make_coords(8, 4, 0.0, 0.0)
    time = syn.make_time(5)
    assert syn.lit_lane_steps(time, x, y, altitude_threshold=-90.0) == (40, 40)  # 8 lanes x 5 steps
    assert syn.lit_lane_steps(time, x, y, altitude_threshold=90.0)[0] == 0
