"""ctypes driver for tests/support/libhost_core.so (1-lane host emulation of the CUDA solver core).

TEST INFRASTRUCTURE ONLY: lets the CPU-only test tier check the kernel's arithmetic against the
oracle.  The product package never loads this library.
"""
import ctypes as C
import os
import re
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
MAX_NCX, MAX_NCU = 4, 8


class FtocpConst(C.Structure):
    _fields_ = [("Q2", C.c_double * 36), ("Qf2", C.c_double * 36), ("R2", C.c_double * 4),
                ("qx", C.c_double * 6), ("qxN", C.c_double * 6), ("dR2", C.c_double * 2),
                ("qs2", C.c_double), ("ql", C.c_double),
                ("Fx", C.c_double * (MAX_NCX * 6)), ("bx", C.c_double * MAX_NCX),
                ("Fu", C.c_double * (MAX_NCU * 2)), ("bu", C.c_double * MAX_NCU),
                ("T", C.c_double * 36), ("Tinv", C.c_double * 36),
                ("eps_res", C.c_double), ("eps_gap", C.c_double), ("d4_min", C.c_double), ("eps_step", C.c_double),
                ("max_iter", C.c_int), ("pad_", C.c_int)]


def make_const(p, Qts=None, eps_res=1e-9, eps_gap=1e-11, d4_min=1e-6, max_iter=40, eps_step=1e-7):
    """p: any object with the reference's MPCParams field names."""
    c = FtocpConst()
    Q, R, Qf = np.asarray(p.Q, float), np.asarray(p.R, float), np.asarray(p.Qf, float)
    xRef = np.asarray(p.xRef, float).ravel()
    c.Q2[:] = (2 * Q).ravel()
    c.Qf2[:] = (2 * Qf).ravel()
    c.R2[:] = (2 * R).ravel()
    c.qx[:] = -2 * Q @ xRef
    c.qxN[:] = -2 * Qf @ xRef
    c.dR2[:] = 2 * np.asarray(p.dR, float).ravel()
    c.qs2, c.ql = 2.0 * float(p.Qslack[0]), float(p.Qslack[1])
    Fx, Fu = np.asarray(p.Fx, float), np.asarray(p.Fu, float)
    fx = np.zeros(MAX_NCX * 6); fx[:Fx.size] = Fx.ravel()
    fu = np.zeros(MAX_NCU * 2); fu[:Fu.size] = Fu.ravel()
    bx = np.zeros(MAX_NCX); bx[:Fx.shape[0]] = np.asarray(p.bx, float).ravel()
    bu = np.zeros(MAX_NCU); bu[:Fu.shape[0]] = np.asarray(p.bu, float).ravel()
    c.Fx[:], c.Fu[:], c.bx[:], c.bu[:] = fx, fu, bx, bu
    T = 2 * np.asarray(Qts, float) if Qts is not None else np.eye(6)
    c.T[:] = T.ravel()
    c.Tinv[:] = np.linalg.inv(T).ravel()
    c.eps_res, c.eps_gap, c.d4_min, c.max_iter, c.eps_step = eps_res, eps_gap, d4_min, max_iter, eps_step
    return c


def pack_abc(A, B, Cc, N):
    A = np.asarray(A, float)
    if A.ndim == 2:
        A = np.tile(A, (N, 1, 1)); B = np.tile(np.asarray(B, float), (N, 1, 1)); Cc = np.zeros((N, 6))
    out = np.zeros((N, 54))
    out[:, 0:36] = np.asarray(A).reshape(N, 36)
    out[:, 36:48] = np.asarray(B).reshape(N, 12)
    out[:, 48:54] = np.asarray(Cc).reshape(N, 6)
    return out


_LAUNCH = os.path.join(_HERE, "..", "..", "racinglmpc_b200", "csrc", "ftocp_launch.cuh")


def kernel_grid():
    """The (N, M) pairs the QP kernel is instantiated for: LMPC_FOR_EACH_CASE of ftocp_launch.cuh, in its order."""
    src = open(_LAUNCH).read()
    body = re.search(r"#define LMPC_FOR_EACH_CASE\(X\)((?:[^\n]*\\\n)*[^\n]*)", src).group(1)
    return [(int(n), int(m)) for n, m in re.findall(r"X\((\d+),\s*(\d+)\)", body)]


_LIBS = {}


def lib(count=False):
    """The host emulation, built on first use.  count=True: a separately named build with -DLMPC_HOST_COUNT that also exports
    host_core_counts (see counts()); its arithmetic is the same."""
    if count not in _LIBS:
        so = os.path.join(_HERE, "libhost_core_count.so" if count else "libhost_core.so")
        src = os.path.join(_HERE, "host_core.cpp")
        hdr = os.path.join(_HERE, "..", "..", "racinglmpc_b200", "csrc", "ftocp_pdip.cuh")
        if (not os.path.exists(so)) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
            flags = ["-DLMPC_HOST_COUNT"] if count else []
            subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas"] + flags + ["-o", so, src],
                           check=True)
        L = C.CDLL(so)
        assert L.host_core_const_size() == C.sizeof(FtocpConst)
        _LIBS[count] = L
    return _LIBS[count]


def counts(reset=True):
    """Branch counts of the counting build since the last reset: dict of corrector passes, recentring passes, step reductions."""
    out = np.zeros(3, np.int64)
    lib(count=True).host_core_counts(out.ctypes.data_as(C.POINTER(C.c_long)), int(reset))
    return dict(corrector=int(out[0]), recentre=int(out[1]), reduce=int(out[2]))


def solve(const, N, abc, x0, uOld, SS=None, Qfun=None, warm=None, count=False):
    """warm: None, or a dict {"buf": float64[>= 512], "valid": int32[1]} carried from solve to solve (the controller's warm-start record).
    count: solve with the counting build (lib(count=True)).  late: 1 when the solve was accepted by the 1e-6 safety net."""
    M = 0 if SS is None else SS.shape[1]
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    abc = np.ascontiguousarray(abc, float)
    ss = np.ascontiguousarray(SS if SS is not None else np.zeros((6, 1)), float)
    qf = np.ascontiguousarray(Qfun if Qfun is not None else np.zeros(1), float)
    x0 = np.ascontiguousarray(x0, float); uOld = np.ascontiguousarray(np.asarray(uOld, float).ravel())
    xp, up = np.zeros((N + 1, 6)), np.zeros((N, 2))
    lam, slack, info = np.zeros(max(M, 1)), np.zeros(N * 2), np.zeros(6)
    wb = None if warm is None else dp(warm["buf"])
    wv = None if warm is None else warm["valid"].ctypes.data_as(C.POINTER(C.c_int))
    rc = lib(count).host_core_solve(N, M, C.byref(const), dp(abc), dp(ss), dp(qf), dp(x0), dp(uOld), dp(xp), dp(up), dp(lam), dp(slack), dp(info), wb, wv)
    assert rc != -1, "unsupported (N, M)"
    return dict(x=xp, u=up, lam=lam[:M], s=slack.reshape(N, 2), status=int(info[0]), iters=int(info[1]),
                r_prim=info[2], r_dual=info[3], gap=info[4], late=int(info[5]))


def warm_point(const, N, M, abc, x0, record):
    """The starting point Pdip::warm_point builds from a warm-start record (float64[>= WS_SIZE]) for the QP (abc, x0):
    dict of x[N+1,6], u[N,2], s, nu1, nu3 [N*2], nu2 [N*4] and, with a safe set, lam, nu4 [M], y1; plus ws_size."""
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    abc = np.ascontiguousarray(abc, float); x0 = np.ascontiguousarray(x0, float); rec = np.ascontiguousarray(record, float)
    R1, R2 = 2 * N, 4 * N                         # the emulation is built for ncx = 2, ncu = 4
    out = np.zeros((N + 1) * 6 + N * 2 + 3 * R1 + R2 + 2 * M + 1)
    n = lib().host_core_warm_point(N, M, C.byref(const), dp(abc), dp(x0), dp(rec), dp(out))
    assert n != -1, "unsupported (N, M)"
    parts, o = {}, 0
    for name, size in (("x", (N + 1) * 6), ("u", N * 2), ("s", R1), ("nu1", R1), ("nu3", R1), ("nu2", R2)) + \
            ((("lam", M), ("nu4", M), ("y1", 1)) if M > 0 else ()):
        parts[name] = out[o:o + size].copy(); o += size
    parts["x"], parts["u"] = parts["x"].reshape(N + 1, 6), parts["u"].reshape(N, 2)
    parts["ws_size"] = n
    return parts
