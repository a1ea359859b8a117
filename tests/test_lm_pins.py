"""The device Levenberg-Marquardt solves and the log-det greedy selection give, bit for bit, the outputs pinned in
tests/golden/lm_solve_pins.npz (tests/golden/make_lm_golden.py): mloam_odom_solve at free_mask 1, 2 and 3 (converged, capped at
max_iterations, a far start whose steps are rejected, a single plane), mloam_calib_rig on three LiDARs with and without priors, and
good_features' gd selection.  They share csrc/lm.cuh's trust-region policy and Cholesky factors."""
import os

import numpy as np
import pytest

import lm_pins_lib as lpl

pytestmark = pytest.mark.gpu
PINS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lm_solve_pins.npz")


@pytest.fixture(scope="module")
def outputs(ctx):
    return lpl.run_all(ctx)


@pytest.mark.parametrize("name", list(lpl.ODOM) + list(lpl.RIG) + list(lpl.GD))
def test_pinned_bits(outputs, name):
    g = np.load(PINS)
    keys = sorted(k for k in g.files if k.startswith(name + "."))
    assert keys and keys == sorted(k for k in outputs if k.startswith(name + "."))
    assert str(outputs[f"{name}.inputs_sha256"]) == str(g[f"{name}.inputs_sha256"]), "the seeded inputs changed"
    for k in keys:
        got, want = np.asarray(outputs[k]), g[k]
        assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes(), (k, got, want)
