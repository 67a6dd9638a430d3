"""Numpy restatement of the state observer of the device closed loop (observe_kernel in csrc/observer.cuh; DESIGN.md,
"Per-controller state observers").

For one step of a batch it forms x_hat from the state the controllers are given (y), the previous prediction's row 1 and
has_pred, with each controller's (mode, gain) row, and returns x_hat, has_pred after the observer and the reset flags.  Every
operation is one fp64 numpy operation, rounded on its own, as the kernel computes it without contraction.
"""
import numpy as np

FLAG_OBSERVER_RESET = 2048


def wrap_guess_s(guess_s, x_s, L):
    """K2's lap-wrap fix of a guess of s (PC.py:392-393): fmax(guess - L, 0) when guess - x > L / 2, else the guess."""
    g, x, L = np.float64(guess_s), np.float64(x_s), np.float64(L)
    return np.fmax(g - L, np.float64(0.0)) if g - x > L / np.float64(2.0) else g


def observe_one(y, prior, has_pred, mode, gain, L, blend=True):
    """One controller: (x_hat [6], has_pred after the observer, reset flag set).  ``prior`` is row 1 of xPredPrev, ``blend`` is
    False for a PID step or a rollout step of mode 2."""
    y = np.asarray(y, np.float64)
    x = y.copy()
    if int(mode) != 1:
        return x, int(has_pred), False
    if not blend:
        return x, 0, False
    if not has_pred:
        return x, int(has_pred), False
    g = np.asarray(gain, np.float64)
    p = np.asarray(prior, np.float64).copy()
    p[4] = wrap_guess_s(p[4], y[4], L)
    if any(g[j] != 1.0 and not np.isfinite(p[j]) for j in range(6)):
        return x, int(has_pred), True
    for j in range(6):
        if g[j] == 1.0:
            continue
        x[j] = p[j] if g[j] == 0.0 else p[j] + g[j] * (y[j] - p[j])
    return x, int(has_pred), False


def observe(y, prior, has_pred, modes, gains, L, blend=True):
    """A batch: y [B, 6], prior [B, 6] (row 1 of xPredPrev), has_pred [B], modes [B], gains [B, 6], L scalar or [B].  Returns
    (x_hat [B, 6], has_pred [B] after the observer, flags [B] with FLAG_OBSERVER_RESET where the prior was reset)."""
    y = np.asarray(y, np.float64)
    B = y.shape[0]
    Ls = np.broadcast_to(np.asarray(L, np.float64), (B,))
    xh = np.zeros_like(y)
    hp = np.zeros(B, np.int32)
    fl = np.zeros(B, np.int32)
    for b in range(B):
        xh[b], hp[b], r = observe_one(y[b], prior[b], has_pred[b], modes[b], gains[b], Ls[b], blend)
        fl[b] = FLAG_OBSERVER_RESET if r else 0
    return xh, hp, fl
