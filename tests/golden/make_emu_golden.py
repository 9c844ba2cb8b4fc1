"""Regenerates tests/golden/emu_outputs_golden.npz (run from the repo root): the emulated kernel's outputs, cold
and then warm, on the instances of tests/test_emu_golden_outputs.py. A reorganisation of the ADMM iteration that
keeps every operation (stage order, where an intermediate lives, which loads are batched) must reproduce them bit
for bit; regenerate them only for a change that is meant to alter the arithmetic."""
import os
import sys

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _ROOT)
from path_optimizer_2_b200 import abi, synthetic  # noqa: E402
from tests.emu import emu  # noqa: E402

# (label, seed, batch, n, ragged, p, reserved bits): n = 63 in both forms (C = 2), n = 120 at C = 4, 128 / 240 / 255
# at C = 8; reserved 32 selects the increment form where it is not the default
CASES = [
    ("n63", 11, 2, 63, False, None, 32),
    ("n63_textbook", 11, 2, 63, False, None, 0),
    ("n120", 12, 2, 120, False, None, 0),
    ("n128_ragged", 13, 2, 128, True, None, 0),
    ("n240", 14, 2, 240, False, None, 0),
    ("n240_rough", 15, 2, 240, False, (70, 0), 0),
    ("n255_ragged", 16, 2, 255, True, None, 0),
]
FIELDS = ("sol", "cost", "status", "iters", "info")


def batch_for(seed, batch, n, ragged, p):
    hb = synthetic.make_batch(seed, batch, n, ragged=ragged)
    if p is not None:
        hb.p = np.array(p, dtype=np.int32)
    return hb


def run_case(seed, batch, n, ragged, p, reserved):
    """Emulated outputs of a capped cold solve and the warm re-solve from its solution."""
    params = abi.default_params(max_iter=50, reserved=reserved)
    hb = batch_for(seed, batch, n, ragged, p)
    es = emu.EmuSolver(params, n, batch)
    cold = es.solve(hb, full=False)
    warm = es.resolve(hb.with_linearisation(cold.sol), full=False)
    out = {}
    for tag, r in (("cold", cold), ("warm", warm)):
        for f in FIELDS:
            out[tag + "_" + f] = np.array(getattr(r, f))
        # the FP32 kernel's solution widened to FP64: stored narrowed again, which is exact
        sol32 = r.sol.astype(np.float32)
        assert np.array_equal(sol32.astype(np.float64), r.sol)
        out[tag + "_sol"] = sol32
    return out


if __name__ == "__main__":
    arrays = {}
    for label, *case in CASES:
        for key, v in run_case(*case).items():
            arrays[label + "/" + key] = v
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu_outputs_golden.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, len(arrays), "arrays")
