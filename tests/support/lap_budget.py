"""Host restatement of the progress numbers (lmpc_rollout_stats / lmpc_rollout_group_stats) under lap budgets
(lmpc_rollout_set_lap_budget)."""
import numpy as np

INT32_MAX = 2 ** 31 - 1


def retired(lap_n, budget):
    """bool [B]: the one rule every kernel uses -- a budget is installed and the controller has handed over that many laps."""
    lap_n = np.asarray(lap_n).reshape(-1)
    return np.zeros(lap_n.shape, bool) if budget is None else lap_n >= np.asarray(budget).reshape(-1)


def group_stats(lap_n, cl_len, flags_or, grp, G, budget=None):
    """[G, 4] int64: (min laps driven over the live controllers, max laps driven over all, min steps into the lap among the live
    controllers at the minimum, controllers with a health flag) of each group; a group without a live controller reports
    (INT32_MAX, lap_max, INT32_MAX, flagged), lap_max and flagged being 0 for a group without controllers."""
    lap_n, cl_len, flags_or, grp = (np.asarray(a).reshape(-1) for a in (lap_n, cl_len, flags_or, grp))
    live = ~retired(lap_n, budget)
    out = np.empty((G, 4), np.int64)
    for g in range(G):
        sel = grp == g
        out[g, 1] = lap_n[sel].max() if sel.any() else 0
        out[g, 3] = int((flags_or[sel] != 0).sum())
        if (sel & live).any():
            out[g, 0] = lap_n[sel & live].min()
            out[g, 2] = cl_len[sel & live & (lap_n == out[g, 0])].min()
        else:
            out[g, 0] = out[g, 2] = INT32_MAX
    return out
