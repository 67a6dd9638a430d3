"""CPU tier: per-controller QP parameters (lmpc_set_param_sets).  The Python-side checks and packing of
_native.make_param_sets, and the host emulation of the solver core on configs[1] QPs under several tunings against the oracle's
assembly of each tuning's QP -- the assembly the GPU tests of heterogeneous batches (test_gpu_param_sets.py) compare against."""
import copy
import ctypes as C
import numpy as np
import pytest
import hostcore as hc
from oracle import ftocp, kkt, osqp_port
from racinglmpc_b200 import _native as nat, workloads, reference_params as rp

B, N = 32, 12


def _base():
    return nat.make_params(rp.mpc_params(N))


def test_library_exports_set_param_sets():
    assert "lmpc_set_param_sets" in nat.exported_symbols()
    assert hasattr(nat.lib(), "lmpc_set_param_sets")


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1),
                                   np.full(B, 0.5)])
def test_bad_index_is_a_value_error(index):
    with pytest.raises(ValueError):
        nat.make_param_sets(_base(), [rp.mpc_params(N), rp.mpc_params(N)], index, B)


def _changed(**kw):
    p = rp.mpc_params(N)
    for k, v in kw.items():
        setattr(p, k, v)
    return p


@pytest.mark.parametrize("bad", [
    dict(N=14),
    dict(Fx=np.array([[0., 0, 0, 0, 0, 1]]), bx=np.array([2.0])),                                 # one lane row
    dict(Fu=np.eye(2), bu=np.array([0.5, 10.0])),                                                 # two input rows
    dict(slacks=False),
    dict(n=5),
    dict(d=3),
])
def test_structural_mismatch_is_a_value_error(bad):
    with pytest.raises(ValueError):
        nat.make_param_sets(_base(), [rp.mpc_params(N), _changed(**bad)], np.arange(B) % 2, B)


def test_no_sets_or_too_many_sets_is_a_value_error():
    with pytest.raises(ValueError):
        nat.make_param_sets(_base(), [], np.zeros(B, int), B)
    with pytest.raises(ValueError):
        nat.make_param_sets(_base(), [rp.mpc_params(N)] * (B + 1), np.zeros(B, int), B)
    _, _, _, _, Qts, lp = rp.lmpc_params(N)
    lbase = nat.make_params(lp, 48, 4, Qts)
    with pytest.raises(ValueError):                                     # one QterminalSlack per set
        nat.make_param_sets(lbase, [lp, lp], np.arange(B) % 2, B, 48, 4, [Qts])


def test_valid_sets_pack_like_make_params():
    _, _, _, _, Qts, lp = rp.lmpc_params(N)
    base = nat.make_params(lp, 48, 4, Qts, eps_res=1e-8, max_iter=30, warm_start=True)
    sets, qts = [], []
    for k in range(5):
        p = copy.deepcopy(lp)
        p.Qslack = np.array([5.0 + k, 25.0 * (k + 1)])
        p.dR = (k + 1) * np.array([1.0, 10.0])
        p.xRef = np.array([0.1 * k, 0, 0, 0, 0, 0])
        sets.append(p)
        qts.append((100.0 + 50 * k) * np.eye(6))
    idx = (7 * np.arange(B)) % 5
    packed, pidx = nat.make_param_sets(base, sets, idx, B, 48, 4, qts)
    assert len(packed) == 5 and pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    for k in range(5):
        ref = nat.make_params(sets[k], 48, 4, qts[k], 1e-8, 0.0, 30, 0.0, warm_start=True)
        assert C.string_at(C.addressof(packed[k]), C.sizeof(nat.Params)) == C.string_at(C.addressof(ref), C.sizeof(nat.Params))
    # None: every set takes the handle's QterminalSlack
    packed, _ = nat.make_param_sets(base, sets, idx, B, 48, 4, None)
    assert all(np.array_equal(np.ctypeslib.as_array(packed[k].QterminalSlack), np.ctypeslib.as_array(base.QterminalSlack))
               for k in range(5))


def mpc_tunings(K=6):
    """configs[1] tunings that differ in every numeric field the QP reads: Q, R, dR, Qslack, xRef, bx, bu."""
    _, base = ftocp.mpc_params(6, 2, N, 0.8)
    base.timeVarying = True
    out = []
    for k in range(K):
        p = copy.deepcopy(base)
        p.Q = np.diag([1.0 + 0.5 * k, 1.0, 1, 1, 0.0, 100.0 / (k + 1)])
        p.R = np.diag([1.0 + k, 10.0 / (k + 1)])
        p.dR = 0.3 * k * np.array([1.0, 10.0])
        p.Qslack = np.array([0.5 * k, 50.0 * (k + 1)])
        p.xRef = np.array([0.6 + 0.1 * k, 0, 0, 0, 0, 0])
        p.bx = np.array([[1.5 + 0.2 * k], [1.5 + 0.2 * k]])
        p.bu = np.array([[0.3 + 0.05 * k], [0.3 + 0.05 * k], [5.0 + k], [5.0 + k]])
        out.append(p)
    return out


def test_host_emulation_of_each_tuning_matches_the_oracle_assembly():
    x0, uold, abc = workloads.ltv_mpc_batch(4, N=N)
    for k, p in enumerate(mpc_tunings()):
        c = hc.make_const(p)
        F, bb = ftocp.build_ineq(p)
        for b in range(3):
            sol = hc.solve(c, N, abc[b], x0[b], uold[b])
            assert sol["status"] == 1, (k, b, sol["status"])
            A = abc[b][:, 0:36].reshape(N, 6, 6); Bm = abc[b][:, 36:48].reshape(N, 6, 2); Cc = abc[b][:, 48:54]
            H, q = ftocp.build_cost(p, uold[b])
            G, E, L = ftocp.build_eq(p, list(A), list(Bm), list(Cc))
            P, q, Am, l, u = ftocp.osqp_form(H, q, F, bb, G, E @ x0[b] + L)
            z, _ = osqp_port.tight_qp(P, q, Am, l, u)
            n = 6 * (N + 1)
            assert np.max(np.abs(sol["x"].ravel() - z[:n])) < 1e-6, (k, b)
            assert np.max(np.abs(sol["u"].ravel() - z[n:n + 2 * N])) < 1e-6, (k, b)
            zz = np.concatenate([sol["x"].ravel(), sol["u"].ravel(), sol["s"].ravel()])
            y = kkt.dual_from_primal(P, q, Am, l, u, zz, tol=1e-6)
            r = kkt.residuals(P, q, Am, l, u, zz, y)
            assert r["r_prim"] < 1e-6 and r["r_dual"] < 1e-6, (k, b, r)


def test_index_is_required_with_params():
    with pytest.raises(ValueError):
        nat.make_param_sets(_base(), [rp.mpc_params(N)], None, B)

