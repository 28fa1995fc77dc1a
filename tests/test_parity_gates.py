"""The parity gates of tests/helpers.py reject what a broken kernel typically returns: a NaN from unwritten or
uninitialised memory, or an infinity, where the reference holds a finite value."""
import numpy as np
import pytest

import helpers as h


@pytest.mark.parametrize("bad_value", [np.nan, np.inf, -np.inf])
def test_gates_reject_non_finite_entries(bad_value):
    ref = np.linspace(-2.0, 3.0, 12).reshape(3, 4)
    mine = ref.copy()
    mine[1, 2] = bad_value
    with pytest.raises(AssertionError, match=r"1/12 outside .* worst at \(.*1.*2.*\)"):
        h.assert_close(mine, ref, what="logits")
    with pytest.raises(AssertionError, match="1/12 outside"):
        h.assert_grad_parity(mine, ref, ref + 1e-3, what="grad")


def test_gates_accept_identical_non_finite_entries():
    ref = np.array([1.0, np.nan, np.inf, -np.inf])
    h.assert_close(ref.copy(), ref)
    h.assert_close(np.zeros(0), np.zeros(0))
