"""Per-controller regression sets in the tests (lmpc_set_regression_sets).

``set_of(group)`` is the regression set a knn_fixtures group was built for.  ``scaled(group, k)`` is the same group with its
scaling and bandwidth multiplied by 2^k: every exact distance, every fp32 partial distance of K1's scan, G, qsum, the threshold
and h scale by 2^k exactly (no rounding changes in the normal range), the weights (1 - (d / h)^2) 3/4 are unchanged bit for bit,
so the pre-filter takes the same decisions at the same margins and the regression computes the same model.  LOW and HIGH are
the exponents of the tests: HIGH puts the unit scaling entries on 2^32, the top of the range the library admits; LOW = -28 is
the lowest power of two that keeps the 0.1 entry of the reference's scaling (0.1 2^-28 = 1.6 2^-32) inside it.
"""
import dataclasses

from racinglmpc_b200.reference_params import RegressionParams

LOW, HIGH = -28, 32


def set_of(group):
    c = group.consts
    return RegressionParams(int(group.trToUse), int(c["MaxNumPoint"]), float(c["h"]), float(c["lamb"]), tuple(c["scaling"]))


def scaled(group, k):
    f = 2.0 ** k
    c = dict(group.consts, h=group.consts["h"] * f, scaling=tuple(s * f for s in group.consts["scaling"]))
    return dataclasses.replace(group, name="%s_x2^%d" % (group.name, k), consts=c)
