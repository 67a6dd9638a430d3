"""CPU tier: the adversarial fixtures of the k-NN regression kernel (tests/support/knn_fixtures.py) do what they are for.

Each fixture must reach the pre-filter branch it was built for, with every decision of the emulated fp32 scan at least 2^-20
(relative) from flipping, so that the double rounding of the emulation cannot change the answer; its exact selection must be
among the candidates the scan hands to the exact re-scoring; the reference must raise where the kernel is to flag; and a fixture
that tests the selection must discriminate: the model of the nearest wrong selection is at least 1000 x the GPU test's tolerance
away from the true model."""
import numpy as np
import pytest

import knn_fixtures as kf

FIXTURES = kf.all_fixtures()
IDS = ["%s/%s" % (g.name, fx.name) for g, fx in FIXTURES]


@pytest.mark.parametrize("case", range(len(FIXTURES)), ids=IDS)
def test_fixture_reaches_its_branch_with_margin(case):
    g, fx = FIXTURES[case]
    laps = kf.used_laps(fx, g.trToUse)
    worst, seen = np.inf, set()
    for i in range(g.N):
        q5 = kf.query(fx, i)
        sel = None
        if not fx.raises:
            m = kf.exact_model(fx, g, exact=False)
            m.model(fx.xLin[i], fx.uLin[i])
            sel = m.last_indices
        for c, (x, u) in enumerate(laps):
            p = kf.prefilter(x, u, q5, g.consts)
            seen.add(p.branch)
            worst = min(worst, kf.min_margin(p))
            if fx.branch[i] is not None:
                assert p.branch == fx.branch[i], (fx.name, i, c, p.branch, p.margins)
            assert kf.min_margin(p) >= kf.MARGIN, (fx.name, i, c, p.margins)
            if sel is not None and p.branch != "overflow":
                # the certified selection: every row the reference picks was re-scored
                assert set(np.atleast_1d(sel[c]).tolist()) <= set(p.cand.tolist()), (fx.name, i, c)
    print("%-40s branches %-28s margin %.2e" % (fx.name, ",".join(sorted(seen)), worst))
    expect_overflow = bool(fx.flags & 32)
    assert ("overflow" in seen) == expect_overflow, (fx.name, seen)


@pytest.mark.parametrize("case", [j for j, (_, fx) in enumerate(FIXTURES) if fx.raises], ids=[IDS[j] for j, (_, fx) in enumerate(FIXTURES) if fx.raises])
def test_reference_raises_where_the_kernel_flags(case):
    g, fx = FIXTURES[case]
    m = kf.exact_model(fx, g, exact=False)
    for i in range(g.N):
        with pytest.raises(fx.raises):
            m.model(fx.xLin[i], fx.uLin[i])


@pytest.mark.parametrize("case", [j for j, (_, fx) in enumerate(FIXTURES) if fx.discriminate],
                         ids=[IDS[j] for j, (_, fx) in enumerate(FIXTURES) if fx.discriminate])
def test_fixture_discriminates_wrong_selections(case):
    g, fx = FIXTURES[case]
    factors = []
    for i in range(g.N):
        m = kf.exact_model(fx, g)
        m.model(fx.xLin[i], fx.uLin[i])
        tol, _ = kf.tolerance(m.systems)
        f = kf.discrimination(fx, g, i, tol)
        if np.isfinite(f):
            factors.append(f)
    print("%-40s discrimination %.1e over %d queries" % (fx.name, min(factors) if factors else np.nan, len(factors)))
    assert factors, "no wrong selection applies to %s" % fx.name
    assert min(factors) >= 1000.0, (fx.name, factors)


def _lost(mutation):
    """{fixture: query-laps whose exact selection is not among the candidates of a pre-filter weakened by `mutation`}."""
    out = {}
    for g, fx in FIXTURES:
        if fx.flags:
            continue
        laps = kf.used_laps(fx, g.trToUse)
        n = 0
        for i in range(g.N):
            m = kf.exact_model(fx, g, exact=False)
            m.model(fx.xLin[i], fx.uLin[i])
            for c, (x, u) in enumerate(laps):
                p = kf.prefilter(x, u, kf.query(fx, i), g.consts, **mutation)
                n += not set(np.atleast_1d(m.last_indices[c]).tolist()) <= set(p.cand.tolist())
        if n:
            out[fx.name] = n
    return out


@pytest.mark.parametrize("mutation, must_catch", [
    (dict(c_abs=0.0), ["magnitude_margin"]),                      # thr without its (G + 2 qsum) 1.3e-6 term
    (dict(recollect=False), ["lane_packing"]),                    # the fast path even when a lane list is full
], ids=["no_rounding_term", "no_recollect"])
def test_a_weakened_prefilter_loses_selected_rows(mutation, must_catch):
    """The margin and the re-collect are not decoration: without either, rows the reference selects are never re-scored."""
    lost = _lost(mutation)
    print("weakened pre-filter %s loses selected rows in: %s" % (mutation, lost))
    for name in must_catch:
        assert lost.get(name, 0) > 0, (mutation, lost)


@pytest.mark.parametrize("case", [j for j, (_, fx) in enumerate(FIXTURES) if fx.kappa],
                         ids=[IDS[j] for j, (_, fx) in enumerate(FIXTURES) if fx.kappa])
def test_conditioning_fixtures_reach_their_condition_numbers(case):
    """kappa_2 of the Gram matrices: the median within half a decade of the target, the largest above it for the targets above
    1e6 (those are bounded by the kappa rule of the GPU test, not by 1e-9)."""
    g, fx = FIXTURES[case]
    ks = []
    for i in range(g.N):
        m = kf.exact_model(fx, g)
        m.model(fx.xLin[i], fx.uLin[i])
        ks.append(max(s[0] for s in m.systems))
    med = float(np.median(ks))
    print("%-24s kappa_2 median %.1e max %.1e (target %.0e)" % (fx.name, med, max(ks), fx.kappa))
    assert abs(np.log10(med / fx.kappa)) <= 0.5, (med, fx.kappa)
    if fx.kappa > 1e6:
        assert max(ks) >= fx.kappa, (max(ks), fx.kappa)


def test_negative_scaling_means_its_absolute_value_in_the_reference():
    g = [g for g in kf.groups() if g.name == "negative_scaling"][0]
    fx = g.fixtures[0]
    pos = dict(g.consts, scaling=tuple(abs(v) for v in g.consts["scaling"]))
    for i in range(3):
        a = kf.ExactLTVModel(kf.TRACK, 1, g.consts, exact=False)
        b = kf.ExactLTVModel(kf.TRACK, 1, pos, exact=False)
        for x, u in fx.laps:
            a.addTrajectory(x, u); b.addTrajectory(x, u)
        ra, rb = a.model(fx.xLin[i], fx.uLin[i]), b.model(fx.xLin[i], fx.uLin[i])
        assert all(np.array_equal(p, q) for p, q in zip(ra, rb))
