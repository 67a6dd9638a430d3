"""CPU tier: warm-started solves of the QP kernel (lmpc_params.warm_start: Pdip::warm_snapshot, Pdip::warm_point and the restart
inside Pdip::solve, racinglmpc_b200/csrc/ftocp_pdip.cuh) through the 1-lane host emulation, QP by QP.

The QPs come in the order a controller meets them (tests/golden/warm_sequences.npz, tests/golden/make_warm_sequences.py): MPC-type
chains at N = 6, 12, 24, 48 whose x0 follows the previous optimum, half of them with jumps in x0, then the same QPs with every
record carried to another chain's model (the largest jump there is), and an LMPC-type sequence at (N, M) = (12, 48) from the
oracle closed loop through a lap crossing.  Each QP is solved cold and warm (one record carried
from solve to solve), and
  - every change of the record's valid flag is one the rule allows (tests/support/warm_record.py), and a solve that finds no usable
    record (valid 0 or 9) is bit for bit the cold solve;
  - the shifted starting point equals a NumPy restatement of it, the 25 % slack floor included;
  - a warm solve is solved wherever the cold one is, at max_iter 40, 24, 20 and 12 -- a restarted solve keeps the cold start's
    budget (below 16 the restart comes at max_iter);
  - every solve that is not a late accept lands within 1e-6 of the oracle's optimum (osqp_port.tight_qp, stored in the fixture)
    or, on LMPC-type QPs, satisfies the KKT conditions of the oracle-assembled QP (and is within 1e-6 wherever the oracle converged).
Late accepts (solved by the 1e-6 safety net, not at eps_res / eps_gap) are counted, never compared with one another."""
import functools
import os
import numpy as np
import pytest
import hostcore as hc
import warm_record as wr
from oracle import ftocp
from racinglmpc_b200 import reference_params as rp

GOLD = os.path.join(os.path.dirname(__file__), "golden")
MPC_N = (6, 12, 24, 48)
MAX_ITERS = (40, 24, 20, 12)
EPS_RES, EPS_GAP = 1e-9, 1e-11


@functools.lru_cache(maxsize=None)
def _fixtures():
    return np.load(os.path.join(GOLD, "warm_sequences.npz")), np.load(os.path.join(GOLD, "workload_ltv.npz"))


def _rollout(abc, x0, u):
    N = u.shape[0]
    x = np.zeros((N + 1, 6)); x[0] = x0
    for k in range(N):
        x[k + 1] = abc[k, 0:36].reshape(6, 6) @ x[k] + abc[k, 36:48].reshape(6, 2) @ u[k] + abc[k, 48:54]
    return x


def _sequences(kind):
    """[(N, M, [qp, ...])]: one list per chain, qp = dict(abc, x0, uold, SS, Qfun, xopt, uopt)"""
    seq, w = _fixtures()
    if kind == "lmpc":
        qps = [dict(abc=seq["lmpc_abc"][k], x0=seq["lmpc_x0"][k], uold=seq["lmpc_uold"][k], SS=seq["lmpc_SS"][k],
                    Qfun=seq["lmpc_Qfun"][k], uopt=seq["lmpc_uopt"][k]) for k in range(seq["lmpc_x0"].shape[0])]
        out = [(12, 48, qps)]
    else:
        N = int(kind)
        out = []
        for ch, start in enumerate(seq["N%d_start" % N]):
            abc = w["N%d_abc" % N][start]
            out.append((N, 0, [dict(abc=abc, x0=seq["N%d_x0" % N][ch, k], uold=seq["N%d_uold" % N][ch, k], SS=None, Qfun=None,
                                    uopt=seq["N%d_uopt" % N][ch, k]) for k in range(seq["N%d_x0" % N].shape[1])]))
        # the same QPs once more, step k of every chain in turn: each record is carried to another model and another x0
        out.append((N, 0, [qps[k] for k in range(len(out[0][2])) for _, _, qps in list(out)]))
    for N, M, qps in out:
        for q in qps:
            q["xopt"] = _rollout(q["abc"], q["x0"], q["uopt"])
    return out


@functools.lru_cache(maxsize=None)
def _const(M, N, max_iter):
    if M > 0:
        _, _, _, _, Qts, lp = ftocp.lmpc_params(_track(), N)
        return hc.make_const(lp, Qts, max_iter=max_iter)
    return hc.make_const(rp.mpc_params(N), max_iter=max_iter)


@functools.lru_cache(maxsize=None)
def _track():
    from oracle.track import TrackTable
    return TrackTable(0.4)


@functools.lru_cache(maxsize=None)
def _run(kind, max_iter):
    """Every QP of the sequences of `kind` solved cold and warm: [dict(N, M, qp, cold, warm, v_in, v_out, record)]"""
    rows = []
    for N, M, qps in _sequences(kind):
        c = _const(M, N, max_iter)
        warm = {"buf": np.zeros(4096), "valid": np.zeros(1, np.int32)}
        for q in qps:
            v_in, rec_in = int(warm["valid"][0]), warm["buf"].copy()
            cold = hc.solve(c, N, q["abc"], q["x0"], q["uold"], q["SS"], q["Qfun"])
            ws = hc.solve(c, N, q["abc"], q["x0"], q["uold"], q["SS"], q["Qfun"], warm=warm)
            rows.append(dict(N=N, M=M, qp=q, cold=cold, warm=ws, v_in=v_in, v_out=int(warm["valid"][0]), record=rec_in))
    return rows


def _late(sol):
    return sol["status"] == 1 and (max(sol["r_prim"], sol["r_dual"]) > EPS_RES * 1.000001 or sol["gap"] > EPS_GAP * 1.000001)


KINDS = [str(n) for n in MPC_N] + ["lmpc"]


@pytest.mark.parametrize("max_iter", MAX_ITERS)
@pytest.mark.parametrize("kind", KINDS)
def test_record_life_cycle_follows_the_rule(kind, max_iter):
    """Every (valid before, valid after) of a solve is a transition the rule allows, and a solve that finds no usable record (valid
    0: none, 9: carried through 8 solves) is the cold solve bit for bit: iterations, status, residuals and every output double."""
    for r in _run(kind, max_iter):
        w, cold = r["warm"], r["cold"]
        assert r["v_out"] in wr.allowed(r["v_in"], w["status"], w["iters"], max_iter), (kind, r["v_in"], r["v_out"], w["status"], w["iters"])
        if not wr.warm_started(r["v_in"]):
            for k in ("status", "iters", "r_prim", "r_dual", "gap"):
                assert w[k] == cold[k], (kind, r["v_in"], k, w[k], cold[k])
            for k in ("x", "u", "lam", "s"):
                assert np.array_equal(w[k], cold[k]), (kind, r["v_in"], k)


def test_record_life_cycle_is_covered():
    """The sequences reach every branch of the rule: ages up to 8 used, an age-9 record re-anchored by a cold start, and
    restarts (a warm start not through by iteration min(16, max_iter)) at every max_iter."""
    seen = {}
    for kind in KINDS:
        for mi in MAX_ITERS:
            for r in _run(kind, mi):
                seen.setdefault((r["v_in"], r["v_out"]), 0)
                seen[(r["v_in"], r["v_out"])] += 1
    assert (8, 9) in seen and (9, 1) in seen, sorted(seen)
    for mi in MAX_ITERS:
        restarts = [r for kind in KINDS for r in _run(kind, mi) if wr.warm_started(r["v_in"]) and r["warm"]["iters"] >= wr.restart_it(mi)]
        assert len(restarts) >= 10 and max(r["cold"]["iters"] for r in restarts) > min(16, mi - 1), (mi, len(restarts))
    print("record transitions (valid before, after): count", dict(sorted(seen.items())))


@pytest.mark.parametrize("max_iter", MAX_ITERS)
def test_warm_solves_are_solved_where_cold_ones_are(max_iter):
    """A warm start that is not through by iteration 16 restarts cold inside the call; the restarted solve gets the full max_iter
    of the cold start it replaces, so it is solved whenever the cold solve is.  Among the restarted QPs at max_iter 40 is one whose
    cold solve needs more than 24 iterations (the budget a restart used to leave)."""
    bad, restarted = [], []
    for kind in KINDS:
        for i, r in enumerate(_run(kind, max_iter)):
            if r["cold"]["status"] == 1 and r["warm"]["status"] != 1:
                bad.append((kind, i, r["v_in"], r["cold"]["iters"], r["warm"]["status"], r["warm"]["iters"]))
            if wr.warm_started(r["v_in"]) and r["warm"]["iters"] >= wr.restart_it(max_iter):
                restarted.append(r["cold"]["iters"])
                assert r["warm"]["iters"] <= max_iter + wr.restart_it(max_iter)
    assert not bad, bad
    assert len(restarted) >= 10, sorted(restarted)
    if max_iter < 40:        # QPs that a restart with max_iter - 16 iterations left could not finish (max_iter 40: the hard pair)
        assert max(restarted) > max_iter - wr.restart_it(max_iter), sorted(restarted)


def test_a_restarted_solve_keeps_the_cold_budget():
    """The stored hard pair (N = 48): a record taken on the first QP is a poor start for the second, whose cold solve needs more
    than 24 iterations.  The warm solve restarts at iteration 16 and, with max_iter 40 of its own, ends solved -- a restart
    that kept only max_iter - 16 iterations ran out.  Both solves are late accepts (residuals and gap <= 1e-6 at iteration
    38, not at eps_res / eps_gap), which bounds the residuals rather than the distance: they are within 1e-5 of the oracle."""
    seq, w = _fixtures()
    N = 48
    abc = w["N%d_abc" % N][int(seq["hard%d_start" % N])]
    c = _const(0, N, 40)
    warm = {"buf": np.zeros(4096), "valid": np.zeros(1, np.int32)}
    hc.solve(c, N, abc, seq["hard%d_x0" % N][0], seq["hard%d_uold" % N][0], warm=warm)
    assert int(warm["valid"][0]) == 1
    x0, uold = seq["hard%d_x0" % N][1], seq["hard%d_uold" % N][1]
    cold = hc.solve(c, N, abc, x0, uold)
    ws = hc.solve(c, N, abc, x0, uold, warm=warm)
    assert cold["status"] == 1 and cold["iters"] > 24, (cold["status"], cold["iters"])
    assert ws["status"] == 1 and wr.RESTART_IT + cold["iters"] == ws["iters"] and int(warm["valid"][0]) == 0, (ws["status"], ws["iters"])
    xopt = _rollout(abc, x0, seq["hard%d_uopt" % N])
    for s in (cold, ws):
        assert np.abs(s["x"] - xopt).max() < 1e-5 and np.abs(s["u"] - seq["hard%d_uopt" % N]).max() < 1e-5
    # the restart is the cold start it replaces, RESTART_IT iterations later: the same iterate
    assert np.array_equal(ws["x"], cold["x"]) and np.array_equal(ws["u"], cold["u"])


def _lmpc_qp(q):
    """The QP of an LMPC-type fixture entry as the oracle assembles it (the reference's code path): OSQP form (P, q, A, l, u)"""
    from oracle import ftocp
    _, _, _, _, Qts, lp = ftocp.lmpc_params(_track(), 12)
    lp.timeVarying = True
    abc = q["abc"]
    A = abc[:, 0:36].reshape(12, 6, 6); B = abc[:, 36:48].reshape(12, 6, 2); C = abc[:, 48:54]
    F, bb = ftocp.build_ineq(lp)
    G, E, L = ftocp.build_eq(lp, list(A), list(B), list(C)); H, qq = ftocp.build_cost(lp, q["uold"][None, :])
    F2, b2, G2, E2, L2, H2, q2 = ftocp.add_safe_set(F, bb, G, E, L, H, qq, 6, 12, q["SS"], q["Qfun"], Qts)
    return ftocp.osqp_form(H2, q2, F2, b2, G2, E2 @ q["x0"] + L2)


@pytest.mark.parametrize("kind", KINDS)
def test_answers_match_the_oracle(kind):
    """Cold and warm solves at the default max_iter; late accepts are counted and printed, every other solve is checked:
    - MPC type: within 1e-6 of the oracle's optimum (osqp_port.tight_qp, DESIGN's parity bar);
    - LMPC type: the point (x, u, s, lambda, terminal slack) satisfies the KKT conditions of the QP the oracle assembles
      (oracle/kkt.py, multipliers fitted to the point) to 1e-8, and is within 1e-6 of the oracle's optimum wherever that optimum
      is itself a KKT point to 1e-9.  On a few QPs just before the finish line OSQP stops (unpolished) with a dual residual of
      ~3e-7 and lands 3e-6 .. 8e-6 from the kernel's answer, whose KKT residuals are ~1e-12 there; those are counted.
    Where neither solve is a late accept, cold and warm agree to 1e-8."""
    from oracle import kkt, osqp_port
    late = {"cold": 0, "warm": 0}
    n, oracle_unconverged = 0, 0
    for r in _run(kind, 40):
        q = r["qp"]
        if kind == "lmpc":
            P, qv, Am, l, u = _lmpc_qp(q)
            zo, _, yo = osqp_port.solve(P, qv, Am, l, u, eps_abs=1e-9, eps_rel=1e-9, max_iter=400000, polish_strict=1)
            ro = kkt.residuals(P, qv, Am, l, u, zo, yo)
            oracle_ok = max(ro["r_prim"], ro["r_dual"], ro["r_comp"]) <= 1e-9
            oracle_unconverged += 0 if oracle_ok else 1
        for which in ("cold", "warm"):
            s = r[which]
            assert s["status"] == 1, (kind, which, s["status"], s["iters"])
            if _late(s):
                late[which] += 1
                continue
            err = max(np.abs(s["x"] - q["xopt"]).max(), np.abs(s["u"] - q["uopt"]).max())
            if kind == "lmpc":
                z = np.concatenate([s["x"].ravel(), s["u"].ravel(), s["s"].ravel(), s["lam"], q["SS"] @ s["lam"] - s["x"][-1]])
                y = kkt.dual_from_primal(P, qv, Am, l, u, z, tol=1e-6)
                rk = kkt.residuals(P, qv, Am, l, u, z, y)
                assert max(rk["r_prim"], rk["r_dual"], rk["r_comp"]) < 1e-8, (which, r["v_in"], rk)
                assert err < 1e-6 or not oracle_ok, (which, r["v_in"], s["iters"], err)
            else:
                assert err < 1e-6, (kind, which, r["v_in"], s["iters"], err)
            n += 1
        if not (_late(r["cold"]) or _late(r["warm"])):
            assert max(np.abs(r["cold"]["x"] - r["warm"]["x"]).max(), np.abs(r["cold"]["u"] - r["warm"]["u"]).max()) < 1e-8
    print("%s: %d solves checked, late accepts cold %d warm %d, oracle optima that are not KKT points to 1e-9: %d" %
          (kind, n, late["cold"], late["warm"], oracle_unconverged))


def _shifted_point(c, N, M, abc, x0, rec):
    """NumPy restatement of Pdip::warm_point: stage k takes stage k+1 and the last stage repeats for u, s, nu1, nu2, nu3 (and the
    derived slack w1 the floor refers to); lam, nu4, y1 are copied; states are rolled out from x0; a derived slack below
    THETA times its old value is lifted to it through the lane slack."""
    R1, R2 = 2 * N, 4 * N
    WS_S = 2 * N; WS_W1 = WS_S + R1; WS_N1 = WS_W1 + R1; WS_N3 = WS_N1 + R1; WS_N2 = WS_N3 + R1; WS_LAM = WS_N2 + R2
    WS_N4 = WS_LAM + M; WS_Y1 = WS_N4 + M

    def shift(a, width):
        a = a.reshape(N, width)
        return np.concatenate([a[1:], a[-1:]])
    u = shift(rec[0:2 * N], 2)
    x = _rollout(abc, x0, u)
    Fx, bx = np.array(c.Fx[:12]).reshape(2, 6), np.array(c.bx[:2])
    s_old, w1_old = shift(rec[WS_S:WS_S + R1], 2), shift(rec[WS_W1:WS_W1 + R1], 2)
    fx = x[:N] @ Fx.T - bx
    floor = wr.THETA * w1_old
    bites = s_old - fx < floor
    out = dict(x=x, u=u, s=np.where(bites, fx + floor, s_old).ravel(), nu1=shift(rec[WS_N1:WS_N1 + R1], 2).ravel(),
               nu3=shift(rec[WS_N3:WS_N3 + R1], 2).ravel(), nu2=shift(rec[WS_N2:WS_N2 + R2], 4).ravel())
    if M > 0:
        out.update(lam=rec[WS_LAM:WS_LAM + M], nu4=rec[WS_N4:WS_N4 + M], y1=rec[WS_Y1:WS_Y1 + 1])
    return out, bites.ravel(), WS_Y1 + 2


@pytest.mark.parametrize("kind", KINDS)
def test_shifted_start_point_matches_numpy(kind):
    """The iterate warm_point builds from the records the sequences carried, and from the same records with the derived slacks
    of alternate rows inflated tenfold (the floor bites there), against the NumPy restatement: copied and shifted values exactly,
    rolled-out states and floored slacks to rounding."""
    rng = np.random.default_rng(3)
    bit, total = 0, 0
    for r in _run(kind, 40):
        if not wr.warm_started(r["v_in"]):
            continue
        N, M, q = r["N"], r["M"], r["qp"]
        c = _const(M, N, 40)
        for variant in range(2):
            rec = r["record"].copy()
            if variant == 1:
                WS_W1 = 4 * N
                rows = np.arange(0, 2 * N, 2) + rng.integers(0, 2)
                rec[WS_W1 + rows] *= 10.0
            got = hc.warm_point(c, N, M, q["abc"], q["x0"], rec)
            ref, bites, ws_size = _shifted_point(c, N, M, q["abc"], q["x0"], rec)
            assert got["ws_size"] == ws_size
            for k in ("u", "nu1", "nu3", "nu2") + (("lam", "nu4", "y1") if M > 0 else ()):
                assert np.array_equal(got[k], ref[k]), (kind, k)
            assert np.allclose(got["x"], ref["x"], rtol=1e-13, atol=1e-13), (kind, np.abs(got["x"] - ref["x"]).max())
            assert np.allclose(got["s"], ref["s"], rtol=1e-12, atol=1e-13), (kind, np.abs(got["s"] - ref["s"]).max())
            bit += int(bites.sum()); total += bites.size
    assert 0 < bit < total, (bit, total)
    print("%s: the slack floor bites on %d of %d rows" % (kind, bit, total))


def test_numpy_spec_warm_theta_is_the_kernels():
    """oracle/pdip_model.py's warm start floors derived slacks at the kernel's WARM_THETA."""
    import inspect
    from oracle import pdip_model as pm
    assert inspect.signature(pm.solve).parameters["warm_theta"].default == wr.THETA
    src = open(os.path.join(os.path.dirname(__file__), "..", "racinglmpc_b200", "csrc", "ftocp_pdip.cuh")).read()
    assert "WARM_THETA = %s;" % wr.THETA in src and "WARM_SNAP_MU = %s, WARM_MIN_MU = %s" % (wr.SNAP_MU, wr.MIN_MU) in src
    assert "WARM_MAX_AGE = %d, WARM_MAX_ITERS = %d" % (wr.MAX_AGE, wr.RESTART_IT) in src
