"""Host restatement of the per-group progress numbers (lmpc_rollout_group_stats) and of the readiness rule that rollout_mc
applied inline before sharding.ready_groups existed."""
import numpy as np

INT32_MAX = 2 ** 31 - 1


def group_stats(lap_n, cl_len, flags_or, grp, G):
    """[G, 4] int64: (min laps driven, max laps driven, min steps into the lap among the controllers at the minimum, controllers
    with a health flag) over the controllers of each group; an empty group is (INT32_MAX, 0, INT32_MAX, 0)."""
    lap_n, cl_len, flags_or, grp = (np.asarray(a).reshape(-1) for a in (lap_n, cl_len, flags_or, grp))
    out = np.empty((G, 4), np.int64)
    for g in range(G):
        sel = grp == g
        if not sel.any():
            out[g] = (INT32_MAX, 0, INT32_MAX, 0)
            continue
        mn = lap_n[sel].min()
        out[g] = (mn, lap_n[sel].max(), cl_len[sel & (lap_n == mn)].min(), int((flags_or[sel] != 0).sum()))
    return out


def inline_rule(lap_min, since, next_round, laps, ship_after):
    """The batch readiness expression of rollout_mc (pooled mode)."""
    return bool(next_round < laps and lap_min >= next_round and (lap_min > next_round or since >= ship_after))
