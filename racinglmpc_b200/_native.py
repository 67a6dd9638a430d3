"""ctypes binding of liblmpc_b200.so (C ABI: include/lmpc_b200.h).

There is NO fallback: if the library is missing or no H100-class (sm_90) device is present, importing the
controllers works but constructing one raises (the product path never routes through the CPU oracle).
"""
import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("LMPC_B200_SO", os.path.join(_HERE, "liblmpc_b200.so"))   # override: kernel-variant experiments only

MAX_NCX, MAX_NCU, MAX_SEG = 4, 8, 16


class Params(C.Structure):
    _fields_ = [("N", C.c_int), ("ncx", C.c_int), ("ncu", C.c_int),
                ("Q", C.c_double * 36), ("R", C.c_double * 4), ("Qf", C.c_double * 36),
                ("dR", C.c_double * 2), ("Qslack", C.c_double * 2), ("xRef", C.c_double * 6),
                ("Fx", C.c_double * (MAX_NCX * 6)), ("bx", C.c_double * MAX_NCX),
                ("Fu", C.c_double * (MAX_NCU * 2)), ("bu", C.c_double * MAX_NCU),
                ("numSS_Points", C.c_int), ("numSS_it", C.c_int), ("QterminalSlack", C.c_double * 36),
                ("eps_res", C.c_double), ("eps_gap", C.c_double), ("max_iter", C.c_int), ("warm_start", C.c_int), ("eps_step", C.c_double)]


class ModelParams(C.Structure):
    _fields_ = [("trToUse", C.c_int), ("MaxNumPoint", C.c_int), ("h", C.c_double), ("lamb", C.c_double),
                ("dt", C.c_double), ("scaling", C.c_double * 5), ("nseg", C.c_int),
                ("seg", C.c_double * (MAX_SEG * 3)), ("TrackLength", C.c_double)]


class VehicleParams(C.Structure):
    """lmpc_vehicle_params: the ten constants of Simulator.dynModel (SysModel.py:61-70)."""
    _fields_ = [(f, C.c_double) for f in ("m", "lf", "lr", "Iz", "Df", "Cf", "Bf", "Dr", "Cr", "Br")]


class TrackParams(C.Structure):
    """lmpc_track_params: the [s_start, length, curvature] rows of Map.PointAndTangent and the lap length."""
    _fields_ = [("nseg", C.c_int), ("seg", C.c_double * (MAX_SEG * 3)), ("TrackLength", C.c_double)]


class NativeError(RuntimeError):
    pass


_LIB = None
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_vp = C.c_void_p


def lib():
    """Load the CUDA library; raise loudly when it is absent."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(_SO):
        raise NativeError("racinglmpc_b200: %s not found — run `python -c \"import __graft_entry__ as g; g.build()\"` "
                          "(nvcc, sm_90a).  There is no CPU fallback." % _SO)
    L = C.CDLL(_SO)
    L.lmpc_last_error.restype = C.c_char_p
    L.lmpc_device_count.restype = C.c_int
    L.lmpc_create.argtypes = [C.POINTER(Params), C.c_int, C.c_int, C.POINTER(_vp)]
    L.lmpc_destroy.argtypes = [_vp]
    L.lmpc_sync.argtypes = [_vp]
    L.lmpc_stream.argtypes = [_vp]
    L.lmpc_stream.restype = _vp
    L.lmpc_kernel_launches.argtypes = [_vp]
    L.lmpc_kernel_launches.restype = C.c_longlong
    L.lmpc_late_accepts.argtypes = [_vp]
    L.lmpc_late_accepts.restype = C.c_longlong
    L.lmpc_set_param_sets.argtypes = [_vp, C.POINTER(Params), C.c_int, _vp]
    ll = C.c_longlong
    for name in ("lmpc_solve_mpc_host", "lmpc_solve_mpc_dev"):
        getattr(L, name).argtypes = [_vp, _vp, _vp, _vp, ll, ll, _vp, _vp, _vp, _vp, _vp, _vp]
    for name in ("lmpc_solve_lmpc_host", "lmpc_solve_lmpc_dev"):
        getattr(L, name).argtypes = [_vp, _vp, _vp, _vp, ll, ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]
    L.lmpc_solve_mpc_host_async.argtypes = [_vp, C.c_int, _vp, _vp, _vp, ll, ll, _vp, _vp, _vp, _vp, _vp, _vp]
    L.lmpc_solve_lmpc_host_async.argtypes = [_vp, C.c_int, _vp, _vp, _vp, ll, ll] + [_vp] * 14
    L.lmpc_host_wait.argtypes = [_vp, C.c_int]
    L.lmpc_host_chunks.argtypes = [_vp, C.c_int]
    ip = C.POINTER(C.c_int)
    L.lmpc_store_create.argtypes = [_vp, C.POINTER(ModelParams), C.c_int, C.c_int, C.c_int]
    L.lmpc_model_put_lap.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp]
    L.lmpc_model_set_used.argtypes = [_vp, _vp]
    L.lmpc_ss_put_lap.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp]
    L.lmpc_ss_set_selection.argtypes = [_vp, _vp, _vp, _vp]
    L.lmpc_ss_add_point.argtypes = [_vp, _vp, _vp]
    L.lmpc_ss_get_lap.argtypes = [_vp, C.c_int, C.c_int, ip, _vp, _vp, _vp]
    L.lmpc_ss_patch_row.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, C.c_int]
    L.lmpc_state_set.argtypes = [_vp] + [_vp] * 7
    L.lmpc_state_get.argtypes = [_vp] + [_vp] * 5
    L.lmpc_identify_host.argtypes = [_vp, _vp, _vp]
    L.lmpc_select_host.argtypes = [_vp] + [_vp] * 7
    L.lmpc_step_host.argtypes = [_vp, C.c_int] + [_vp] * 11
    L.lmpc_step_dev.argtypes = [_vp, C.c_int, _vp]
    L.lmpc_step_profile.argtypes = [_vp, C.c_int, _vp, _vp]
    L.lmpc_step_results.argtypes = [_vp, _vp, _vp, _vp, _vp]
    L.lmpc_read_buffer.argtypes = [_vp, C.c_char_p, C.c_size_t, _vp, C.c_size_t]
    L.lmpc_device_buffer.argtypes = [_vp, C.c_char_p]
    L.lmpc_device_buffer.restype = _vp
    L.lmpc_rollout_create.argtypes = [_vp, C.c_int]
    L.lmpc_rollout_set_state.argtypes = [_vp, _vp, _vp]
    L.lmpc_rollout_get_state.argtypes = [_vp, _vp, _vp, _vp, _vp]
    L.lmpc_rollout_step.argtypes = [_vp, C.c_int, _vp, C.c_ulonglong]
    L.lmpc_rollout_get_health.argtypes = [_vp, _vp, _vp]
    L.lmpc_rollout_pid_step.argtypes = [_vp, C.c_double, _vp, _vp, C.c_ulonglong]
    L.lmpc_rollout_set_vehicles.argtypes = [_vp, C.POINTER(VehicleParams), C.c_int, _vp]
    L.lmpc_set_tracks.argtypes = [_vp, C.POINTER(TrackParams), C.c_int, _vp]
    L.lmpc_rollout_sysid.argtypes = [_vp, C.c_double, _vp, _vp]
    L.lmpc_rollout_seed_from_record.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.lmpc_rollout_get_lap.argtypes = [_vp, C.c_int, ip, _vp, _vp]
    L.lmpc_rollout_commit_lap.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.lmpc_rollout_commit_laps.argtypes = [_vp, _vp, _vp, _vp]
    L.lmpc_rollout_export_laps_dev.argtypes = [_vp, C.c_int, _vp, _vp]
    L.lmpc_ss_export_laps_dev.argtypes = [_vp, _vp, C.c_int, _vp, _vp]
    L.lmpc_ss_import_laps_dev.argtypes = [_vp, _vp, _vp, _vp, C.c_int, C.c_int, _vp, _vp]
    L.lmpc_probe_fp64.argtypes = [C.c_int, _vp]
    L.lmpc_track_global_position.argtypes = [C.c_int, _vp, C.c_int, C.c_double, C.c_int, _vp, _vp, _vp, _vp]
    L.lmpc_rollout_trace_create.argtypes = [_vp, C.c_int, _vp, C.c_int]
    L.lmpc_rollout_trace_get.argtypes = [_vp, C.c_int, _vp] + [_vp] * 6
    L.lmpc_books_set.argtypes = [_vp] * 7
    L.lmpc_books_get.argtypes = [_vp] * 13
    L.lmpc_rollout_commit_laps_dev.argtypes = [_vp]
    L.lmpc_rollout_seed_from_record_dev.argtypes = [_vp, C.c_int]
    L.lmpc_rollout_stats.argtypes = [_vp, _vp]
    L.lmpc_pool_export_dev.argtypes = [_vp, C.c_int, C.c_int, C.c_longlong, _vp, _vp]
    L.lmpc_pool_import_dev.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_longlong, _vp, _vp, _vp]
    L.lmpc_host_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(_vp)]
    L.lmpc_host_free.argtypes = [_vp]
    L.lmpc_host_numa_node.argtypes = [C.c_int]
    L.lmpc_host_page_nodes.argtypes = [_vp, C.c_size_t, C.c_int, _vp]
    L.lmpc_sizeof_params.restype = C.c_int
    L.lmpc_sizeof_model_params.restype = C.c_int
    L.lmpc_sizeof_vehicle_params.restype = C.c_int
    L.lmpc_sizeof_track_params.restype = C.c_int
    assert L.lmpc_sizeof_params() == C.sizeof(Params), "lmpc_params ABI mismatch"
    assert L.lmpc_sizeof_model_params() == C.sizeof(ModelParams), "lmpc_model_params ABI mismatch"
    assert L.lmpc_sizeof_vehicle_params() == C.sizeof(VehicleParams), "lmpc_vehicle_params ABI mismatch"
    assert L.lmpc_sizeof_track_params() == C.sizeof(TrackParams), "lmpc_track_params ABI mismatch"
    _LIB = L
    return L


def make_model_params(seg_table, TrackLength, trToUse, MaxNumPoint=7, h=5.0, lamb=0.0, dt=0.1,
                      scaling=(0.1, 1.0, 1.0, 1.0, 1.0)):
    """PredictiveModel.__init__ constants (PredictiveModel.py:12-32) + the track's [s0, length, curvature] rows."""
    m = ModelParams()
    m.trToUse, m.MaxNumPoint = int(trToUse), int(MaxNumPoint)
    m.h, m.lamb, m.dt = float(h), float(lamb), float(dt)
    m.scaling[:] = list(scaling)
    seg = np.asarray(seg_table, float).reshape(-1, 3)
    if seg.shape[0] > MAX_SEG:
        raise ValueError("track table has more than %d segments" % MAX_SEG)
    m.nseg = seg.shape[0]
    buf = np.zeros(MAX_SEG * 3)
    buf[:seg.size] = seg.ravel()
    m.seg[:] = buf
    m.TrackLength = float(TrackLength)
    return m


def check(rc):
    if rc != 0:
        raise NativeError("liblmpc_b200 error %d: %s" % (rc, lib().lmpc_last_error().decode()))


def probe_fp64(device=0):
    """Measured fp64 numbers of the device (csrc/probe.cuh): the roofline denominators of the QP kernel."""
    out = np.zeros(8)
    check(lib().lmpc_probe_fp64(int(device), out.ctypes.data_as(_vp)))
    keys = ("dfma_tflops", "dmma_tflops", "lat_dfma", "lat_dmma_acc", "lat_dmma_a", "lat_lds", "lat_shfl64", "lat_rsqrt")
    return dict(zip(keys, (float(v) for v in out)))


class _PinnedBlock:
    """Owner of one lmpc_host_alloc block; freed when the last ndarray viewing it dies."""

    def __init__(self, device, nbytes):
        p = _vp()
        check(lib().lmpc_host_alloc(int(device), max(int(nbytes), 1), C.byref(p)))
        self.ptr, self.nbytes = p.value, int(nbytes)

    def __del__(self):
        try:
            if self.ptr:
                lib().lmpc_host_free(_vp(self.ptr))
                self.ptr = None
        except Exception:
            pass


def pinned_empty(shape, dtype=np.float64, device=0):
    """Zero-filled C-contiguous ndarray in pinned host memory on the device's NUMA node (lmpc_host_alloc): the
    buffers to hand to the ``*_host`` / ``solve_async`` entry points."""
    dt = np.dtype(dtype)
    n = int(np.prod(shape)) if np.ndim(shape) else int(shape)
    blk = _PinnedBlock(device, n * dt.itemsize)
    buf = (C.c_char * max(n * dt.itemsize, 1)).from_address(blk.ptr)
    a = np.frombuffer(buf, dtype=dt, count=n).reshape(shape)
    buf._lmpc_owner = blk            # ndarray.base -> buf -> blk: the block lives as long as any view of it
    return a


def page_nodes(a, n=8):
    """NUMA node of ``n`` evenly sampled pages of a host ndarray (diagnostics of the pinned allocator)."""
    out = np.zeros(n, np.int32)
    check(lib().lmpc_host_page_nodes(a.ctypes.data_as(_vp), a.nbytes, int(n), out.ctypes.data_as(_vp)))
    return out.tolist()


def pinned_like(a, device=0):
    """Copy of ``a`` (any array-like) in pinned host memory on the device's NUMA node."""
    a = np.asarray(a)
    out = pinned_empty(a.shape, a.dtype, device)
    out[...] = a
    return out


def exported_symbols():
    """Names include/lmpc_b200.h declares; used by the CPU-tier test that the library exports them."""
    hdr = os.path.join(_HERE, "..", "include", "lmpc_b200.h")
    import re
    txt = open(hdr).read()
    return sorted(set(re.findall(r"\b(lmpc_[a-z_0-9]+)\s*\(", txt)))


def ptr(a):
    """Host ndarray / int address / object with data_ptr() -> void*."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(_vp)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    return C.c_void_p(int(a))


def make_params(p, numSS_Points=0, numSS_it=0, QterminalSlack=None, eps_res=0.0, eps_gap=0.0, max_iter=0, eps_step=0.0, warm_start=False):
    """p: object with the reference's MPCParams field names (PredictiveControllers.py:24-51)."""
    if int(p.n) != 6 or int(p.d) != 2:
        raise ValueError("racinglmpc_b200 supports n == 6, d == 2 (the reference's vehicle model)")
    if not bool(p.slacks):
        raise ValueError("racinglmpc_b200 implements the soft-lane formulation (slacks=True) the reference uses")
    q = Params()
    q.N = int(p.N)
    Fx, Fu = np.asarray(p.Fx, float), np.asarray(p.Fu, float)
    q.ncx, q.ncu = Fx.shape[0], Fu.shape[0]
    if q.ncx > MAX_NCX or q.ncu > MAX_NCU:
        raise ValueError("too many constraint rows")
    q.Q[:] = np.asarray(p.Q, float).ravel()
    q.R[:] = np.asarray(p.R, float).ravel()
    q.Qf[:] = np.asarray(p.Qf, float).ravel()
    q.dR[:] = np.asarray(p.dR, float).ravel()
    q.Qslack[:] = np.asarray(p.Qslack, float).ravel()
    q.xRef[:] = np.asarray(p.xRef, float).ravel()
    fx = np.zeros(MAX_NCX * 6); fx[:Fx.size] = Fx.ravel()
    fu = np.zeros(MAX_NCU * 2); fu[:Fu.size] = Fu.ravel()
    bx = np.zeros(MAX_NCX); bx[:q.ncx] = np.asarray(p.bx, float).ravel()
    bu = np.zeros(MAX_NCU); bu[:q.ncu] = np.asarray(p.bu, float).ravel()
    q.Fx[:], q.Fu[:], q.bx[:], q.bu[:] = fx, fu, bx, bu
    q.numSS_Points, q.numSS_it = int(numSS_Points), int(numSS_it)
    q.QterminalSlack[:] = (np.asarray(QterminalSlack, float).ravel() if QterminalSlack is not None else np.zeros(36))
    q.eps_res, q.eps_gap, q.max_iter, q.eps_step = float(eps_res), float(eps_gap), int(max_iter), float(eps_step)
    q.warm_start = 1 if warm_start else 0
    return q


def _set_index(index, K, batch, what):
    """The index rules of the per-controller tables (lmpc_set_param_sets, lmpc_rollout_set_vehicles, lmpc_set_tracks): 1 <= K <= batch rows and
    one integer row number in [0, K) per controller.  Returns the index as a contiguous int32 array; raises ValueError."""
    if index is None:
        raise ValueError("index is required: one set number per controller (%d)" % batch)
    if not 1 <= K <= batch:
        raise ValueError("need 1 .. batch (= %d) %s, got %d" % (batch, what, K))
    idx = np.ascontiguousarray(np.asarray(index).reshape(-1), dtype=np.int32)
    if idx.shape[0] != batch or not np.array_equal(idx, np.asarray(index).reshape(-1)):
        raise ValueError("index must hold one integer set number per controller (%d)" % batch)
    if idx.min() < 0 or idx.max() >= K:
        raise ValueError("set index out of range [0, %d)" % K)
    return idx


def make_param_sets(base, params, index, batch, numSS_Points=0, numSS_it=0, QterminalSlack=None):
    """Per-controller parameters for ``lmpc_set_param_sets``: K MPCParams-like objects ``params``, the set of every controller
    ``index[batch]`` and ``QterminalSlack`` (None: the base's, or one 6x6 matrix per set).  ``base`` is the handle's own ``Params``;
    the interior-point settings (tolerances, max_iter, warm_start) are taken from it.  Each set is converted by ``make_params``.
    Raises ValueError where the library would refuse: an index of the wrong length or out of range, or a set that differs from
    the base in N, the rows of Fx or Fu, slacks or n/d.  Returns (ctypes array Params * K, int32 index array)."""
    params = list(params)
    K = len(params)
    idx = _set_index(index, K, batch, "parameter sets")
    if QterminalSlack is None:
        qts = [np.ctypeslib.as_array(base.QterminalSlack).reshape(6, 6).copy()] * K
    else:
        qts = list(QterminalSlack)
        if len(qts) != K:
            raise ValueError("QterminalSlack needs one matrix per set (%d)" % K)
    out = (Params * K)()
    for k, (p, q) in enumerate(zip(params, qts)):
        s = make_params(p, numSS_Points, numSS_it, q, base.eps_res, base.eps_gap, base.max_iter, base.eps_step, bool(base.warm_start))
        if (s.N, s.ncx, s.ncu) != (base.N, base.ncx, base.ncu):
            raise ValueError("set %d: N / rows of Fx / rows of Fu (%d, %d, %d) differ from the handle's (%d, %d, %d)"
                             % (k, s.N, s.ncx, s.ncu, base.N, base.ncx, base.ncu))
        if (s.numSS_Points, s.numSS_it) != (base.numSS_Points, base.numSS_it):
            raise ValueError("set %d: numSS_Points / numSS_it differ from the handle's" % k)
        out[k] = s
    return out, idx


VEHICLE_FIELDS = tuple(f for f, _ in VehicleParams._fields_)


def make_vehicle_sets(vehicles, index, batch):
    """Per-controller vehicles for ``lmpc_rollout_set_vehicles``: K objects ``vehicles`` with the reference's field names (m, lf,
    lr, Iz, Df, Cf, Bf, Dr, Cr, Br; e.g. reference_params.VehicleParams) and the vehicle of every controller ``index[batch]``.
    Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, a non-positive m, Iz, lf or lr,
    or a value that is not finite.  Returns (ctypes array VehicleParams * K, int32 index array)."""
    vehicles = list(vehicles)
    K = len(vehicles)
    idx = _set_index(index, K, batch, "vehicles")
    out = (VehicleParams * K)()
    for k, v in enumerate(vehicles):
        vals = [float(getattr(v, f)) for f in VEHICLE_FIELDS]
        if not all(np.isfinite(vals)):
            raise ValueError("vehicle %d: every value must be finite" % k)
        if min(v.m, v.Iz, v.lf, v.lr) <= 0:
            raise ValueError("vehicle %d: m, Iz, lf and lr must be positive" % k)
        out[k] = VehicleParams(*vals)
    return out, idx


def make_track_sets(tracks, index, batch):
    """Per-controller tracks for ``lmpc_set_tracks``: K objects ``tracks`` with ``seg_table`` ([nseg, 3] rows s_start, length,
    curvature) and ``TrackLength`` (e.g. reference_params.TrackParams) and the track of every controller ``index[batch]``.
    Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, 1 .. 16 rows, a value that is not
    finite, a negative length, a first start other than 0, a start other than the previous start + length, or a TrackLength that
    is not positive or not the last start + length (all exact: Track.py:54-133 builds the table that way).
    Returns (ctypes array TrackParams * K, int32 index array)."""
    tracks = list(tracks)
    K = len(tracks)
    idx = _set_index(index, K, batch, "tracks")
    out = (TrackParams * K)()
    for k, t in enumerate(tracks):
        seg = np.asarray(t.seg_table, dtype=float)
        L = float(t.TrackLength)
        if seg.ndim != 2 or seg.shape[1] != 3 or not 1 <= seg.shape[0] <= MAX_SEG:
            raise ValueError("track %d: seg_table must have 1 .. %d rows of [s_start, length, curvature]" % (k, MAX_SEG))
        if not (np.all(np.isfinite(seg)) and np.isfinite(L)):
            raise ValueError("track %d: every value must be finite" % k)
        if np.any(seg[:, 1] < 0):
            raise ValueError("track %d: a segment has a negative length" % k)
        if seg[0, 0] != 0.0:
            raise ValueError("track %d: the first segment must start at s = 0" % k)
        for i in range(1, seg.shape[0]):
            if seg[i, 0] != seg[i - 1, 0] + seg[i - 1, 1]:
                raise ValueError("track %d: segment %d does not start where segment %d ends" % (k, i, i - 1))
        if not L > 0 or L != seg[-1, 0] + seg[-1, 1]:
            raise ValueError("track %d: TrackLength must be positive and equal the end of the last segment" % k)
        buf = np.zeros(MAX_SEG * 3)
        buf[:seg.size] = seg.ravel()
        out[k].nseg = seg.shape[0]
        out[k].seg[:] = buf
        out[k].TrackLength = L
    return out, idx
