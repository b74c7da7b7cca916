"""GPU: with the zero-point means accumulated in float64 the solver is expected to reproduce EVERY level of the reference's fixtures
(it does when the kernels' source runs on the emulator, tests/test_emu_cpu.py).  Written after round 1's GPU budget was spent: the
bound the validated suite asserts stays <= 5e-4 (tests/test_quantize_gpu.py); this stricter statement is a non-strict xfail until it
has been seen on the GPU (the SFU's ex2/lg2 only matter for elements whose error survives the shrinkage -- none in these fixtures)."""
import numpy as np
import pytest
import torch

from hqq_b200 import ops

pytestmark = pytest.mark.gpu
COMBOS = [(nbits, axis, gs) for nbits in (8, 4, 3, 2, 1) for axis in (0, 1) for gs in ((64,) if nbits != 4 else (64, 32, 128))]


@pytest.mark.parametrize("nbits,axis,gs", COMBOS)
def test_solver_levels_equal_the_reference_fixtures(golden, oracle, nbits, axis, gs):
    q = golden.quant
    key = f"b{nbits}_a{axis}_g{gs}"
    W = torch.from_numpy(q["W"]).to("cuda:0")
    W_q, scale, zero, tr = ops.quantize(W, nbits=nbits, group_size=gs, axis=axis, round_zero=(nbits == 4), optimize=True, want_trace=True)
    pk = oracle.BIT_TO_PACKING[nbits]
    rows = q["W"].size // gs if axis == 1 else gs
    assert int(tr["info"][0]) == int(q[key + "/iters"])
    assert np.array_equal(oracle.UNPACK[pk](W_q.cpu().numpy())[:rows], oracle.UNPACK[pk](q[key + "/W_q"])[:rows])


@pytest.mark.parametrize("nbits,axis", [(nbits, axis) for nbits in (4, 2, 1) for axis in (0, 1)])
def test_solver_on_heavy_tailed_weights(golden, oracle, nbits, axis):
    """quantize_heavy: the shrinkage's |x|^(p-1) branch is active, i.e. the SFU's ex2 / lg2 take part.  Bound: the validated suite's
    (<= 5e-4 of the levels by one level, stop iteration +-1); on the emulator the kernels reproduce every level."""
    h = golden.heavy
    key = f"b{nbits}_a{axis}_g64"
    W = torch.from_numpy(h["W"]).to("cuda:0")
    W_q, scale, zero, tr = ops.quantize(W, nbits=nbits, group_size=64, axis=axis, round_zero=(nbits == 4), optimize=True, want_trace=True)
    pk = oracle.BIT_TO_PACKING[nbits]
    rows = h["W"].size // 64 if axis == 1 else 64
    a = oracle.UNPACK[pk](W_q.cpu().numpy())[:rows].astype(int)
    b = oracle.UNPACK[pk](h[key + "/W_q"])[:rows].astype(int)
    assert abs(int(tr["info"][0]) - int(h[key + "/iters"])) <= 1
    assert np.abs(a - b).max() <= 1 and (a != b).mean() <= 5e-4
