"""CPU tier: the host emulation of the QP kernel (tests/support/host_core.cpp) over the kernel's whole (N, M) grid, and its
iterates after a few interior-point iterations against the NumPy specification (oracle/pdip_model.py).

The device's tensor-core sweeps are compared with this emulation iteration by iteration in tests/test_gpu_qp_iterates.py.
That comparison cannot see a mistake the two share (starting point, residuals, step rule, termination): the truncated solves
below pin that shared code to the specification, step by step."""
import numpy as np
import pytest

import hostcore as hc
from oracle import pdip_model as pm
from qp_inputs import ltv_inputs, lmpc_qp_inputs
from racinglmpc_b200 import workloads, reference_params as rp


def test_host_emulation_covers_the_kernel_grid(gold):
    """Every (N, M) of LMPC_FOR_EACH_CASE is instantiated in the host emulation and solves a QP of its shape; a pair outside
    the grid is refused (so the two lists cannot drift apart unnoticed)."""
    grid = hc.kernel_grid()
    assert len(grid) == len(set(grid)) == 30, grid
    for N, M in grid:
        if M == 0:
            x0, uold, abc, _ = ltv_inputs(1, N)
            sol = hc.solve(hc.make_const(rp.mpc_params(N)), N, abc[0], x0[0], uold[0])
        else:
            _, _, _, _, Qts, par = rp.lmpc_params(N)
            x0, uold, abc, SS, Qf, _, _ = lmpc_qp_inputs(gold, N, 1, False, M)
            sol = hc.solve(hc.make_const(par, Qts), N, abc[0], x0[0], uold[0], SS[0], Qf[0])
        assert sol["status"] == 1 and sol["late"] == 0, (N, M, sol["status"], sol["iters"])
    with pytest.raises(AssertionError, match="unsupported"):
        hc.solve(hc.make_const(rp.mpc_params(13)), 13, np.zeros((13, 54)), np.zeros(6), np.zeros(2))


@pytest.mark.parametrize("N,B", [(12, 16), (48, 4)])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_truncated_solves_follow_the_numpy_spec(N, B, k):
    """After k iterations (max_iter = k) the host emulation's iterate (x, u, lane slacks), status and iteration count are the
    specification's with the kernel's constants, to 1e-10: the same number of factorisations, the same step on every QP."""
    x0, uold, abc = workloads.ltv_mpc_batch(B, N=N)
    p = rp.mpc_params(N)
    c = hc.make_const(p, max_iter=k)
    for b in range(B):
        A = abc[b][:, 0:36].reshape(N, 6, 6); Bm = abc[b][:, 36:48].reshape(N, 6, 2); C = abc[b][:, 48:54]
        ref = pm.solve(pm.from_params(p, A, Bm, C, x0[b], uold[b]), eps=1e-9, eps_gap=1e-11, max_iter=k,
                       **pm.kernel_constants(N, False))
        sol = hc.solve(c, N, abc[b], x0[b], uold[b])
        assert (sol["status"], sol["iters"], sol["late"]) == (ref["status"], ref["iters"], int(ref["late"])), \
            (N, k, b, sol["status"], sol["iters"], ref["status"], ref["iters"])
        err = max(np.abs(sol["x"] - ref["x"]).max(), np.abs(sol["u"] - ref["u"]).max(), np.abs(sol["s"] - ref["s"]).max())
        assert err < 1e-10, (N, k, b, err)
