"""Batched FTOCP solver front-end: B independent controllers' QPs per launch.

This is the batched counterpart of one ``MPC.solve`` / ``LMPC.solve`` QP hand-off
(src/fnc/controller/PredictiveControllers.py:110-137,259-283): the per-instance data the reference
assembles into (H,q,F,b,G,E,L) is passed as stage data and solved on the GPU by
csrc/lmpc_b200.cu.  Host (NumPy) arrays go through the ``*_host`` C entry points (copies inside);
objects exposing ``data_ptr()`` (torch CUDA tensors) or raw device addresses go through ``*_dev``.
"""
import ctypes as C
import numpy as np
from . import _native as nat


def pack_abc(A, B, Cc=None):
    """[..., N, 6,6], [..., N, 6,2], [..., N, 6] -> [..., N, 54] stage records (A | B | C)."""
    A, B = np.asarray(A, float), np.asarray(B, float)
    lead = A.shape[:-2]
    out = np.zeros(lead + (54,))
    out[..., 0:36] = A.reshape(lead + (36,))
    out[..., 36:48] = B.reshape(lead + (12,))
    if Cc is not None:
        out[..., 48:54] = np.asarray(Cc, float)
    return out


class BatchedFTOCP:
    """``batch`` QPs with identical cost/constraint parameters (an MPCParams-like object), or per-controller parameters after
    ``set_param_sets``."""

    def __init__(self, params, batch, device=0, numSS_Points=0, numSS_it=0, QterminalSlack=None,
                 eps_res=0.0, eps_gap=0.0, max_iter=0):
        L = nat.lib()
        self._lib = L
        self.N, self.B, self.M = int(params.N), int(batch), int(numSS_Points)
        self.ncx = np.asarray(params.Fx).shape[0]
        self.device = device
        self._p = nat.make_params(params, numSS_Points, numSS_it, QterminalSlack, eps_res, eps_gap, max_iter)
        h = C.c_void_p()
        nat.check(L.lmpc_create(C.byref(self._p), self.B, int(device), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.lmpc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def kernel_launches(self):
        return int(self._lib.lmpc_kernel_launches(self._h))

    @property
    def late_accepts(self):
        """QPs accepted at the 1e-6 safety-net tolerance instead of eps_res / eps_gap since creation (expected 0)."""
        return int(self._lib.lmpc_late_accepts(self._h))

    def set_param_sets(self, params, index=None, QterminalSlack=None):
        """Per-controller QP parameters (a parameter sweep in one batch): controller b solves with ``params[index[b]]`` (objects
        with the reference's MPCParams field names; every field but N and the constraint row counts may differ) and, for LMPC,
        ``QterminalSlack[index[b]]`` (None: the handle's).  ``index`` is required with ``params``.  ``params=None`` (no index)
        returns to the parameters the handle was created with.
        Waits for work already enqueued; warm-start records start over."""
        if params is None:
            if index is not None:
                raise ValueError("params=None reverts to the handle's own parameters and takes no index")
            nat.check(self._lib.lmpc_set_param_sets(self._h, None, 0, None))
            return
        sets, idx = nat.make_param_sets(self._p, params, index, self.B, self._p.numSS_Points, self._p.numSS_it, QterminalSlack)
        nat.check(self._lib.lmpc_set_param_sets(self._h, sets, len(sets), nat.ptr(idx)))

    def sync(self):
        nat.check(self._lib.lmpc_sync(self._h))

    # ------------------------------------------------------------------ host arrays
    def _abc_layout(self, abc):
        abc = np.ascontiguousarray(abc, dtype=np.float64)
        N = self.N
        if abc.shape == (self.B, N, 54):
            return abc, N * 54, 54
        if abc.shape == (N, 54):
            return abc, 0, 54
        if abc.shape == (54,):
            return abc, 0, 0
        raise ValueError("abc must be [B,N,54], [N,54] or [54]")

    def solve(self, x0, uOld, abc, SS_sel=None, Qfun_sel=None, Succ_SS=None, Succ_uSS=None, out=None):
        """Host path.  Returns dict of NumPy arrays (allocated once and reused when ``out`` is given)."""
        B, N, M = self.B, self.N, self.M
        f = lambda a, shape: np.ascontiguousarray(np.asarray(a, dtype=np.float64).reshape(shape))
        x0, uOld = f(x0, (B, 6)), f(uOld, (B, 2))
        abc, s_i, s_k = self._abc_layout(abc)
        o = out if out is not None else self.alloc_outputs(SS_sel is not None)
        if SS_sel is None:
            nat.check(self._lib.lmpc_solve_mpc_host(self._h, nat.ptr(x0), nat.ptr(uOld), nat.ptr(abc), s_i, s_k,
                                                    nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["slack"]),
                                                    nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"])))
        else:
            SS_sel, Qfun_sel = f(SS_sel, (B, 6, M)), f(Qfun_sel, (B, M))
            Succ_SS = None if Succ_SS is None else f(Succ_SS, (B, 6, M))
            Succ_uSS = None if Succ_uSS is None else f(Succ_uSS, (B, 2, M))
            nat.check(self._lib.lmpc_solve_lmpc_host(
                self._h, nat.ptr(x0), nat.ptr(uOld), nat.ptr(abc), s_i, s_k, nat.ptr(SS_sel), nat.ptr(Qfun_sel),
                nat.ptr(Succ_SS), nat.ptr(Succ_uSS), nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["slack"]),
                nat.ptr(o["lambd"]), nat.ptr(o["slackTerminal"]), nat.ptr(o["zt"]), nat.ptr(o["zt_u"]),
                nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"])))
        return o

    def solve_async(self, slot, x0, uOld, abc, out, SS_sel=None, Qfun_sel=None, Succ_SS=None, Succ_uSS=None):
        """Enqueue a host-path solve on buffer set ``slot`` (0 .. 3) and return at once; ``wait(slot)`` completes it.
        Every array (inputs and the ``out`` dict of ``alloc_outputs``) must be C-contiguous float64/int32, should be pinned,
        and must stay alive and untouched until the wait.  Two slots in flight overlap the copies of one batch with the solve
        of the other; three keep the copy engine busy across the host's wait / enqueue of the next batch."""
        B, N, M = self.B, self.N, self.M
        for a in (x0, uOld, abc):
            if not (isinstance(a, np.ndarray) and a.flags.c_contiguous and a.dtype == np.float64):
                raise ValueError("solve_async takes C-contiguous float64 arrays (no hidden copies that could die before wait())")
        abc, s_i, s_k = self._abc_layout(abc)
        o = out
        if SS_sel is None:
            nat.check(self._lib.lmpc_solve_mpc_host_async(self._h, int(slot), nat.ptr(x0), nat.ptr(uOld), nat.ptr(abc), s_i, s_k,
                                                          nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["slack"]),
                                                          nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"])))
        else:
            nat.check(self._lib.lmpc_solve_lmpc_host_async(
                self._h, int(slot), nat.ptr(x0), nat.ptr(uOld), nat.ptr(abc), s_i, s_k, nat.ptr(SS_sel), nat.ptr(Qfun_sel),
                nat.ptr(Succ_SS), nat.ptr(Succ_uSS), nat.ptr(o["xPred"]), nat.ptr(o["uPred"]), nat.ptr(o["slack"]),
                nat.ptr(o["lambd"]), nat.ptr(o["slackTerminal"]), nat.ptr(o["zt"]), nat.ptr(o["zt_u"]),
                nat.ptr(o["status"]), nat.ptr(o["iters"]), nat.ptr(o["resid"])))
        return o

    def wait(self, slot):
        nat.check(self._lib.lmpc_host_wait(self._h, int(slot)))

    def alloc_outputs(self, lmpc=False):
        B, N, M = self.B, self.N, max(self.M, 1)
        o = dict(xPred=np.zeros((B, N + 1, 6)), uPred=np.zeros((B, N, 2)), slack=np.zeros((B, N * self.ncx)),
                 status=np.zeros(B, np.int32), iters=np.zeros(B, np.int32), resid=np.zeros((B, 3)))
        if lmpc:
            o.update(lambd=np.zeros((B, M)), slackTerminal=np.zeros((B, 6)), zt=np.zeros((B, 6)), zt_u=np.zeros((B, 2)))
        return o

    # ------------------------------------------------------------------ device pointers
    def solve_dev(self, x0, uOld, abc, abc_inst_stride, abc_stage_stride, xPred, uPred, status, iters, resid,
                  slack=None, SS_sel=None, Qfun_sel=None, Succ_SS=None, Succ_uSS=None, lambd=None,
                  slackTerminal=None, zt=None, zt_u=None):
        """Device path: every argument is a device pointer (int) or an object with ``data_ptr()``.
        Enqueues on the handle's stream; call ``sync()`` before reading results."""
        p = nat.ptr
        if SS_sel is None:
            nat.check(self._lib.lmpc_solve_mpc_dev(self._h, p(x0), p(uOld), p(abc), int(abc_inst_stride),
                                                   int(abc_stage_stride), p(xPred), p(uPred), p(slack), p(status),
                                                   p(iters), p(resid)))
        else:
            nat.check(self._lib.lmpc_solve_lmpc_dev(self._h, p(x0), p(uOld), p(abc), int(abc_inst_stride),
                                                    int(abc_stage_stride), p(SS_sel), p(Qfun_sel), p(Succ_SS),
                                                    p(Succ_uSS), p(xPred), p(uPred), p(slack), p(lambd),
                                                    p(slackTerminal), p(zt), p(zt_u), p(status), p(iters), p(resid)))

    @property
    def stream(self):
        return int(self._lib.lmpc_stream(self._h) or 0)
