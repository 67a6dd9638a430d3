"""The life cycle of a controller's warm-start record (Pdip::solve in racinglmpc_b200/csrc/ftocp_pdip.cuh), restated.
TEST INFRASTRUCTURE ONLY.

valid = 0: no record; 1..MAX_AGE: a record that has been carried through valid - 1 solves -- the solve warm-starts from it;
MAX_AGE + 1: a record too old to use -- the solve starts cold.  A solve snapshots its first iterate with mu <= SNAP_MU and keeps it
only if mu >= MIN_MU.  New valid: old + 1 after a warm start, 1 after a cold start, 0 without a snapshot; 0 after a warm start
that restarted cold or did not end solved.

allowed() checks the valid flag only: a kept snapshot (old + 1 or 1) and none (0) are both allowed after a clean solve, because
the host emulation does not report the gap at which a snapshot was taken -- the snapshot window itself is not checked here."""
SNAP_MU, MIN_MU, THETA = 0.1, 0.01, 0.25
MAX_AGE, RESTART_IT = 8, 16


def warm_started(valid_in):
    return 1 <= valid_in <= MAX_AGE


def restart_it(max_iter):
    """the iteration at which a warm start that is not through restarts cold"""
    return min(RESTART_IT, max_iter)


def allowed(valid_in, status, iters, max_iter):
    """the values the record's valid flag may take after a solve that ended with (status, iters)"""
    if not warm_started(valid_in):
        return {0, 1}
    if iters >= restart_it(max_iter) or status != 1:      # restarted, or not through: the record is dropped
        return {0}
    return {0, valid_in + 1}
