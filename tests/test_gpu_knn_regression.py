"""GPU tier: the k-NN regression kernel (K1) on adversarial neighbourhoods (tests/support/knn_fixtures.py) against an exact
reference: the oracle's selection with ties to the lowest row and the Gram systems solved in mpmath at 60 digits.

Per instance: flags equal the expected bits (0 where the reference computes a model; 1, 2, 4 where it raises; 32 where more rows
lie within fp32 resolution of the k-th neighbour than can be re-scored).  Per query of a clean instance: rows 3..5 within 1e-14 of
the oracle; rows 0..2 within 1e-9 where kappa_2(Q) <= 1e6, else within 32 kappa_2 2^-53 |theta*|_inf."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import knn_fixtures as kf                                           # noqa: E402
from racinglmpc_b200 import reference_params as rp                 # noqa: E402
from racinglmpc_b200.controller import BatchedController          # noqa: E402

GROUPS = kf.groups()


@pytest.mark.parametrize("gi", range(len(GROUPS)), ids=[g.name for g in GROUPS])
def test_k1_matches_the_exact_reference(gi):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    g = GROUPS[gi]
    B = len(g.fixtures)
    c = BatchedController(rp.mpc_params(g.N), B, kf.TRACK.seg_table(), kf.TRACK.TrackLength, trToUse=g.trToUse, Tmax=g.Tmax,
                          model_cap=g.model_cap, model_kwargs=g.consts)
    try:
        for b, fx in enumerate(g.fixtures):
            for x, u in fx.laps:
                c.model_add_trajectory(b, x, u)
        c.set_state(xLin=np.stack([fx.xLin for fx in g.fixtures]), uLin=np.stack([fx.uLin for fx in g.fixtures]),
                    OldInput=np.zeros((B, 2)), timeStep=np.zeros(B))
        abc, flags = c.identify()
    finally:
        c.close()
    assert [int(f) for f in flags] == [fx.flags for fx in g.fixtures], [fx.name for fx in g.fixtures]
    for b, fx in enumerate(g.fixtures):
        if fx.flags:
            continue
        m = kf.exact_model(fx, g)
        rep = []
        for i in range(g.N):
            A, Bm, C = m.model(fx.xLin[i], fx.uLin[i])
            tol, kap = kf.tolerance(m.systems)
            gA, gB, gC = kf.abc_split(abc[b, i])
            err = float(np.max(np.abs(kf.rows012(gA, gB, gC) - kf.rows012(A, Bm, C))))
            err_np = max(float(np.max(np.abs(s[2] - s[1]))) for s in m.systems)
            e345 = float(np.max(np.abs(kf.rows345(gA, gB, gC) - kf.rows345(A, Bm, C))))
            rep.append((kap, err, err_np, tol))
            assert err <= tol, (fx.name, i, "kappa %.2e kernel %.2e np.linalg.solve %.2e tol %.2e" % (kap, err, err_np, tol))
            assert e345 <= 1e-14, (fx.name, i, e345)
        k = max(r[0] for r in rep)
        print("%-36s kappa<=%.1e kernel err %.2e np.linalg.solve err %.2e (tol >= %.1e)" %
              (fx.name, k, max(r[1] for r in rep), max(r[2] for r in rep), min(r[3] for r in rep)))
