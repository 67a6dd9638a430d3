"""GPU tier: the QP kernel's iterates, not only its answers, against the host emulation of the same kernel
(tests/support/host_core.cpp) at every instantiated (N, M).

The device runs the Riccati sweeps on fp64 tensor-core fragments (open-loop sweeps for M > 0, closed-loop sweeps for M = 0,
STREAM sweeps that read the stage model from global memory for N >= 32); the host emulation runs the scalar sweeps of the same
header.  Everything else is shared: starting point, residuals, step rule, termination (pinned to the NumPy specification by
tests/test_qp_iterates.py).  An interior-point method corrects an inexact Newton direction at the price of iterations, so a
wrong gain or cost-to-go entry can still reach the right answer; stopping both after k iterations (max_iter = k) shows it.

  - Truncated solves, every pair: each QP solved on the device and on the host after k in DEPTHS iterations and at the default
    limit.  Per QP and depth: status, iteration count, xPred, uPred, slack (and lambd for M > 0) within TOL, residuals within TOL
    relative to max(1, |host|) (r_dual within rd_tol(M, k)).  A QP "separates" at the first depth where it disagrees.  Rounding can
    flip a step reduction or a recentring decision late in a solve (LP-degenerate QPs one iteration apart), so separation is
    allowed from depth SEP_FROM on, for at most SEP_PAIR of a pair's batch and SEP_ALL of its family; a systematic error
    separates most QPs of a pair at depth 1 (each of four value mutants of the sweeps did, one of them in the
    costate row that only r_dual shows).  Full solves: the same status on every QP,
    iteration counts equal but for ITER_MISMATCH of a pair's QPs (never more than one apart), answers within TOL wherever
    neither solve is a late accept.  The message names the pair and depth.
  - Layout of the stage model (device entry solve_dev): guard stages, a stage stride of 64 doubles and NaN in every padding
    double, per-instance and shared (abc_inst_stride = 0) models, at the staged (N = 12) and STREAM (N = 32, 48) forms: results
    bit-identical to the packed host-entry solve.
  - Branch coverage: the host side counts its corrector passes, recentring passes and step reductions (the counting build of
    the emulation); both families (M = 0 and M > 0) must take recentring passes and step reductions, in the staged and in the
    STREAM form (perturbed QPs screened on the host for a recentring pass are added to the batches), so that the discrete
    decisions device and emulation must agree on are compared.

The kernels for per-controller parameters and per-controller shapes need no run of their own here:
test_gpu_param_sets.py::test_every_instantiation_bit_identical_to_uniform_handles and test_gpu_shape_sets.py pin them bit for
bit to the uniform kernel compared here.
Thresholds: measured on an H100, profiles/h100_qp_iterates.txt."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from racinglmpc_b200 import BatchedFTOCP, reference_params as rp            # noqa: E402
import hostcore as hc                                                       # noqa: E402
from qp_inputs import ltv_inputs, lmpc_qp_inputs, perturbed_lmpc_inputs, perturbed_ltv_inputs   # noqa: E402

# Thresholds from profiles/h100_qp_iterates.txt (H100 80GB HBM3 at 700 W), per family (M = 0 / M > 0), with the margin stated
DEPTHS = (1, 2, 3, 5, 8, 0)          # iteration limits; 0 = the default limit (40)
TOL = 1e-8                           # iterates, r_prim, gap, full-solve answers


def rd_tol(M, k):
    """Tolerance of r_dual (relative to max(1, |host|)) at depth k.  M = 0: TOL at every depth.  With a safe set, r_dual is
    mostly the simplex-row residual Qfun + y1 - nu4 - SS' yT with yT = -T xi, T = 2 QterminalSlack (10^2 .. 10^4 times the
    stage weights), and the rounding of xi grows with |T| while the iterate still agrees to TOL (the profile splits r_dual into
    that part and the input-stationarity part): looser only where those data need it."""
    if M == 0 or k == 0:
        return TOL
    return 1e-3 if k == 8 else 1e-6


SEP_FROM = 5                         # a QP may separate from this depth on: none separated before depth 8
SEP_PAIR = {False: 0.02, True: 0.25}    # separated QPs per pair: at most max(1, SEP_PAIR * batch)
SEP_ALL = {False: 0.005, True: 0.10}    # ... and over the family
ITER_MISMATCH = {False: 0.02, True: 0.25}   # full solves one iteration apart per pair: at most max(1, ITER_MISMATCH * batch)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no GPU")


def _qps(gold, N, M):
    """The QP set of pair (N, M): dict of inputs, the handle's parameters and the host emulation's constants (max_iter aside)."""
    if M == 0:
        par, Qts = rp.mpc_params(N), None
        x0, uold, abc, _ = ltv_inputs(64, N)
        # far from the operating point: 16 of them, and those of 512 that take a recentring pass on the host (none of the 64 do)
        px, pu, pa = perturbed_ltv_inputs(512, N, seed=N)
        c = hc.make_const(par)
        hc.counts()
        pick = list(range(16))
        for b in range(16, 512):
            hc.solve(c, N, pa[b], px[b], pu[b], count=True)
            if hc.counts()["recentre"] and len(pick) < 20:
                pick.append(b)
        hc.counts()
        x0, uold, abc = (np.concatenate([a, p[pick]]) for a, p in ((x0, px), (uold, pu), (abc, pa)))
        return dict(x0=x0, uold=uold, abc=abc, SS=None, Qf=None, par=par, Qts=None, numSS_it=0)
    numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
    parts = [lmpc_qp_inputs(gold, N, 16, dup, M)[:5] for dup in (False, True)]      # duplicated laps: LP-degenerate QPs
    if N >= 32:
        # the STREAM form: those of 512 perturbed QPs that take a recentring pass and solve on the host (none of the 32 do)
        px, pu, pa, pS, pQ = perturbed_lmpc_inputs(gold, N, 512, seed=N, M=M)
        c = hc.make_const(par, Qts)
        hc.counts()
        pick = []
        for b in range(512):
            sol = hc.solve(c, N, pa[b], px[b], pu[b], pS[b], pQ[b], count=True)
            if hc.counts()["recentre"] and sol["status"] == 1 and len(pick) < 4:
                pick.append(b)
        hc.counts()
        parts.append(tuple(a[pick] for a in (px, pu, pa, pS, pQ)))
    if (N, M) == (12, 48):
        # closed-loop QPs on which the solver used to ride the neighbourhood boundary (test_host_core.py): they take the
        # recentring pass
        d = np.load(os.path.join(GOLDEN, "stalled_lmpc_qps.npz"))
        parts.append(tuple(np.stack([d["q%d_%s" % (i, k)] for i in range(8)]) for k in ("x0", "uold", "abc", "SS", "Qf")))
    x0, uold, abc, SS, Qf = (np.ascontiguousarray(np.concatenate(a)) for a in zip(*parts))
    return dict(x0=x0, uold=uold, abc=abc, SS=SS, Qf=Qf, par=par, Qts=Qts, numSS_it=numSS_it)


def _device(q, N, M, max_iter):
    s = BatchedFTOCP(q["par"], batch=q["x0"].shape[0], numSS_Points=M, numSS_it=q["numSS_it"], QterminalSlack=q["Qts"],
                     max_iter=max_iter)
    o = s.solve(q["x0"], q["uold"], q["abc"], q["SS"], q["Qf"])
    o = {k: v.copy() for k, v in o.items()}
    s.close()
    return o


def _host(q, N, M, max_iter):
    c = hc.make_const(q["par"], q["Qts"], max_iter=max_iter or 40)
    out = []
    for b in range(q["x0"].shape[0]):
        args = (c, N, q["abc"][b], q["x0"][b], q["uold"][b]) + ((q["SS"][b], q["Qf"][b]) if M else ())
        out.append(hc.solve(*args, count=True))
    return out


def _late(status, resid):
    return status == 1 and (max(resid[0], resid[1]) > 1.000001e-9 or resid[2] > 1.000001e-11)


def _diff(o, h, b, M):
    """Largest |device - host| of QP b over the iterate; of r_prim and gap, and of r_dual, relative to max(1, |host|)."""
    d = max(np.abs(o["xPred"][b] - h["x"]).max(), np.abs(o["uPred"][b] - h["u"]).max(),
            np.abs(o["slack"][b] - h["s"].ravel()).max())
    if M:
        d = max(d, np.abs(o["lambd"][b] - h["lam"]).max())
    hr = np.array([h["r_prim"], h["r_dual"], h["gap"]])
    rel = np.abs(o["resid"][b] - hr) / np.maximum(1.0, np.abs(hr))
    return d, float(max(rel[0], rel[2])), float(rel[1])


def test_truncated_iterates_match_the_host_emulation_at_every_pair(gold):
    _need_gpu()
    rows, failures = [], []
    # host branch counts per family, and per family in the STREAM form (N >= 32)
    counts = {(fam, st): dict(corrector=0, recentre=0, reduce=0) for fam in (False, True) for st in (False, True)}
    n_all, sep_all = {False: 0, True: 0}, {False: 0, True: 0}
    for N, M in hc.kernel_grid():
        q = _qps(gold, N, M)
        B = q["x0"].shape[0]
        sep_at = np.full(B, -1)                 # index into DEPTHS of the first disagreement
        for di, k in enumerate(DEPTHS):
            o, h = _device(q, N, M, k), _host(q, N, M, k)
            for key, v in hc.counts().items():
                counts[(M > 0, N >= 32)][key] += v
            worst = worst_r = worst_rd = 0.0
            n_it = 0
            for b in range(B):
                d, dr, drd = _diff(o, h[b], b, M)
                same = (o["status"][b] == h[b]["status"] and o["iters"][b] == h[b]["iters"])
                if k == 0:
                    # full solves: status always, iterations nearly always, answers wherever neither solve is a late accept
                    d_it = abs(int(o["iters"][b]) - h[b]["iters"])
                    n_it += d_it != 0
                    hr = (h[b]["r_prim"], h[b]["r_dual"], h[b]["gap"])
                    if o["status"][b] != h[b]["status"] or d_it > 1:
                        failures.append("(N, M) = (%d, %d), full solve, QP %d: status %d / %d, iterations %d / %d (device / host)"
                                        % (N, M, b, o["status"][b], h[b]["status"], o["iters"][b], h[b]["iters"]))
                    elif not (_late(int(o["status"][b]), o["resid"][b]) or _late(h[b]["status"], hr)) and d > TOL:
                        failures.append("(N, M) = (%d, %d), full solve, QP %d: |d answer| %.2e" % (N, M, b, d))
                if sep_at[b] >= 0:
                    continue
                if same and d <= TOL and dr <= TOL and drd <= rd_tol(M, k):
                    worst, worst_r, worst_rd = max(worst, d), max(worst_r, dr), max(worst_rd, drd)
                    continue
                sep_at[b] = di
                if 0 < k < SEP_FROM:
                    failures.append("(N, M) = (%d, %d), depth %d, QP %d: separates from the host emulation (status %d / %d, "
                                    "iterations %d / %d, |d| %.2e, r_prim / gap %.2e, r_dual %.2e)" % (
                                        N, M, k, b, o["status"][b], h[b]["status"], o["iters"][b], h[b]["iters"], d, dr, drd))
            rows.append("N %2d M %2d  B %3d  depth %2s  separated %2d  worst |d| %.2e  r_prim/gap %.2e  r_dual %.2e%s" % (
                N, M, B, k or "40", int(np.sum(sep_at == di)), worst, worst_r, worst_rd,
                ("  full-solve iteration mismatches %d" % n_it) if k == 0 else ""))
            if k == 0 and n_it > max(1, ITER_MISMATCH[M > 0] * B):
                failures.append("(N, M) = (%d, %d), full solve: %d of %d QPs with other iteration counts" % (N, M, n_it, B))
        n_sep = int(np.sum(sep_at >= 0))
        n_all[M > 0] += B
        sep_all[M > 0] += n_sep
        if n_sep > max(1, SEP_PAIR[M > 0] * B):
            first = DEPTHS[int(sep_at[sep_at >= 0].min())] or 40
            failures.append("(N, M) = (%d, %d): %d of %d QPs separate from the host emulation (first at depth %d)" % (N, M, n_sep, B, first))
    print("\n".join(rows))
    for (fam, st), c in counts.items():
        print("host branch counts, %s, %s: %s" % ("M > 0" if fam else "M = 0", "N >= 32" if st else "N < 32", c))
    for fam in (False, True):
        print("%s: separated %d of %d QPs (%.3f %%)" % ("M > 0" if fam else "M = 0", sep_all[fam], n_all[fam],
                                                          100.0 * sep_all[fam] / n_all[fam]))
    assert not failures, "\n".join(failures[:40])
    for fam in (False, True):
        assert sep_all[fam] <= SEP_ALL[fam] * n_all[fam], ("M > 0" if fam else "M = 0", sep_all[fam], n_all[fam])
        # recentring passes and step reductions compared in the staged and in the STREAM form of each family
        for st in (False, True):
            c = counts[(fam, st)]
            assert c["recentre"] > 0 and c["reduce"] > 0, ("M > 0" if fam else "M = 0", "N >= 32" if st else "N < 32", c)


def _padded(abc, shared, N):
    """abc [B, N, 54] in one allocation of NaN: a guard stage before and after each instance's N stages, stage stride 64
    doubles.  Returns (tensor, address of instance 0's stage 0, instance stride, stage stride)."""
    S = 64
    src = torch.from_numpy(abc[0] if shared else abc)
    t = torch.full(((1 if shared else abc.shape[0]), N + 2, S), float("nan"), dtype=torch.float64)
    t[..., 1:N + 1, :54] = src
    t = t.cuda()
    return t, t.data_ptr() + S * 8, (0 if shared else (N + 2) * S), S


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("N,M", [(12, 0), (12, 48), (32, 0), (32, 48), (48, 0), (48, 48)])
def test_strided_stage_model_bit_identical_to_packed(gold, N, M, shared):
    _need_gpu()
    B = 32
    if M == 0:
        par, Qts, numSS_it = rp.mpc_params(N), None, 0
        x0, uold, abc, _ = ltv_inputs(B, N)
        SS = Qf = None
    else:
        numSS_it, _, _, _, Qts, par = rp.lmpc_params(N)
        x0, uold, abc, SS, Qf, _, _ = lmpc_qp_inputs(gold, N, B, False, M)
    s = BatchedFTOCP(par, batch=B, numSS_Points=M, numSS_it=numSS_it, QterminalSlack=Qts)
    ref = s.solve(x0, uold, abc[0] if shared else abc, SS, Qf)
    ref = {k: v.copy() for k, v in ref.items()}
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t, p0, s_i, s_k = _padded(abc, shared, N)
    o = dict(xPred=torch.zeros(B, N + 1, 6, dtype=torch.float64, device="cuda"),
             uPred=torch.zeros(B, N, 2, dtype=torch.float64, device="cuda"),
             slack=torch.zeros(B, 2 * N, dtype=torch.float64, device="cuda"),
             status=torch.zeros(B, dtype=torch.int32, device="cuda"), iters=torch.zeros(B, dtype=torch.int32, device="cuda"),
             resid=torch.zeros(B, 3, dtype=torch.float64, device="cuda"))
    d_x0, d_uold = dev(x0), dev(uold)         # held until after sync(): the kernel reads them on the handle's stream
    kw = {}
    if M:
        o["lambd"] = torch.zeros(B, M, dtype=torch.float64, device="cuda")
        d_SS, d_Qf = dev(SS), dev(Qf)
        kw = dict(SS_sel=d_SS, Qfun_sel=d_Qf, lambd=o["lambd"])
    s.solve_dev(d_x0, d_uold, p0, s_i, s_k, o["xPred"], o["uPred"], o["status"], o["iters"], o["resid"],
                slack=o["slack"], **kw)
    s.sync()
    assert np.all(ref["status"] == 1), ref["status"]
    for k, v in o.items():
        a = v.cpu().numpy()
        assert np.array_equal(a, ref[k]), (N, M, shared, k, np.nanmax(np.abs(a - ref[k])) if a.dtype == np.float64 else None)
    assert torch.isnan(t[..., 54:]).all() and torch.isnan(t[..., 0, :]).all() and torch.isnan(t[..., N + 1, :]).all()
    s.close()
