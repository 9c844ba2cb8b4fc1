"""The emulated kernel reproduces its recorded outputs (tests/golden/make_emu_golden.py) bit for bit: sol, cost,
status, iteration count and info (residual norms, rho, rho updates), cold and then warm, at n = 63 .. 255 on plain,
ragged and rough instances capped at 50 iterations, in the increment and the textbook form. A reorganisation of
the ADMM iteration that keeps every operation must pass unchanged; a reordered or dropped term fails it."""
import os

import numpy as np
import pytest

from tests.golden import make_emu_golden as mk

_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emu_outputs_golden.npz")


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32)


@pytest.mark.parametrize("case", mk.CASES, ids=[c[0] for c in mk.CASES])
def test_emulated_outputs_match_the_recorded_ones_bit_for_bit(case):
    label, *args = case
    golden = np.load(_GOLDEN)
    got = mk.run_case(*args)
    for key, v in got.items():
        want = golden[label + "/" + key]
        assert v.dtype == want.dtype and v.shape == want.shape, key
        assert np.array_equal(_bits(v), _bits(want)), (label, key)
