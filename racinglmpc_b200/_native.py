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
MAX_POOL_GROUPS = 64


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


class NoiseParams(C.Structure):
    """lmpc_noise_params: the clipped Gaussian noise of Simulator.dynModel (SysModel.py:139-145) and of the PID path follower
    (Utilities.py:42-68)."""
    _fields_ = [("sim_sigma", C.c_double * 3), ("sim_clip", C.c_double * 3), ("sim_gain", C.c_double),
                ("pid_sigma", C.c_double * 2), ("pid_clip", C.c_double * 2)]


class MeasurementParams(C.Structure):
    """lmpc_measurement_params: the clipped Gaussian sensor noise on (vx, vy, wz, epsi, s, ey) that the controllers of the device
    closed loop see."""
    _fields_ = [("sigma", C.c_double * 6), ("clip", C.c_double * 6)]


class ObserverParams(C.Structure):
    """lmpc_observer_params: the fixed-gain state observer of a controller of the device closed loop -- mode 0 none, mode 1
    x_hat_j = p_j + gain_j (y_j - p_j) over (vx, vy, wz, epsi, s, ey), p the controller's own one-step prediction."""
    _fields_ = [("mode", C.c_int), ("pad", C.c_int), ("gain", C.c_double * 6)]


class RegressionParams(C.Structure):
    """lmpc_regression_params: the constants of the local regression model (PredictiveModel.py:18-31)."""
    _fields_ = [("trToUse", C.c_int), ("MaxNumPoint", C.c_int), ("h", C.c_double), ("lamb", C.c_double),
                ("scaling", C.c_double * 5)]


class ShapeParams(C.Structure):
    """lmpc_shape_params: the horizon N and the safe-set size numSS_Points of a controller."""
    _fields_ = [("N", C.c_int), ("numSS_Points", C.c_int)]


class SsLapsParams(C.Structure):
    """lmpc_ss_laps_params: numSS_it, the number of fastest past laps a controller's safe set draws from."""
    _fields_ = [("numSS_it", C.c_int)]


class LapWindowParams(C.Structure):
    """lmpc_lap_window_params: the most recent laps a controller's safe set (ss_window) and learned model (model_window) draw
    from; 0 = unbounded."""
    _fields_ = [("ss_window", C.c_int), ("model_window", C.c_int)]


class LaneRuleParams(C.Structure):
    """lmpc_lane_rule_params: mode 0 ranks laps by lap time (the reference's rule), mode 1 ranks a lap that left the lane by more
    than lane_tol behind every lap that kept to it."""
    _fields_ = [("mode", C.c_int), ("pad", C.c_int), ("lane_tol", C.c_double)]


class LaneMarginParams(C.Structure):
    """lmpc_lane_margin_params: the margin a controller's QPs narrow its lane by -- mode 0 none, mode 1 margin0, mode 2 adapted
    lap by lap within [margin0, margin_max] (step_up after a lap that left the lane, step_down after one that kept to it)."""
    _fields_ = [("mode", C.c_int), ("pad", C.c_int), ("margin0", C.c_double), ("margin_max", C.c_double), ("step_up", C.c_double),
                ("step_down", C.c_double)]


class PredictionModelParams(C.Structure):
    """lmpc_prediction_model_params: where rows 0..2 of a controller's LTV model come from -- mode 0 the k-NN regression (the
    reference), mode 1 the exact linearisation of ``vehicle``, mode 2 that of the plant's own vehicle row."""
    _fields_ = [("mode", C.c_int), ("pad", C.c_int), ("vehicle", VehicleParams)]


class ObserverGainParams(C.Structure):
    """lmpc_observer_gain_params: the gains a mode 1 observer blends with -- mode 0 its row's fixed gains, mode 1 the frozen-time
    Kalman gain of the linearised car for the diagonal process covariance ``q`` (per control period) and measurement covariance
    ``r`` over (vx, vy, wz, epsi, s, ey)."""
    _fields_ = [("mode", C.c_int), ("pad", C.c_int), ("q", C.c_double * 6), ("r", C.c_double * 6)]


class ObserverPriorParams(C.Structure):
    """lmpc_observer_prior_params: where a mode 1 observer takes its prior from -- source 0 its own plan, source 1 the
    simulator's noise-free control period for ``vehicle``, source 2 that of the plant's own vehicle and surface rows."""
    _fields_ = [("source", C.c_int), ("pad", C.c_int), ("vehicle", VehicleParams)]


MAX_ZONES = 16                      # LMPC_MAX_ZONES: zones of one track-surface row


class SurfaceParams(C.Structure):
    """lmpc_surface_params: nzone friction zones (s_start, s_end, mu_f, mu_r) along the lap; a sub-step whose wrapped s lies in
    [s_start, s_end) of a zone drives with peak tyre forces mu_f Df and mu_r Dr."""
    _fields_ = [("nzone", C.c_int), ("pad", C.c_int), ("zone", C.c_double * (MAX_ZONES * 4))]


FLAG_NOMINAL_NONFINITE = 1024       # LMPC_FLAG_NOMINAL_NONFINITE: step flag of a nominal controller whose rows 0..2 are not finite
FLAG_OBSERVER_RESET = 2048          # LMPC_FLAG_OBSERVER_RESET: step flag of an observer whose prior was not finite (it read y)
FLAG_OBSERVER_GAIN = 4096           # LMPC_FLAG_OBSERVER_GAIN: step flag of an observer whose model gain could not be formed (it read y)
LANE_UNSAFE_KEY = 1 << 24           # LMPC_LANE_UNSAFE_KEY: added to the safe-set key of a lane-unsafe lap
REPORT_LANE_UNSAFE = 1 << 16        # LMPC_REPORT_LANE_UNSAFE: report flag of an own lap judged lane-unsafe


def split_lane_key(ss_time):
    """(lap time, unsafe) of safe-set keys (``books()["ss_time"]``, a scalar or an array): a key >= LANE_UNSAFE_KEY is a lap judged
    lane-unsafe under a lane rule, filed as lap time + LANE_UNSAFE_KEY.  A free slot's key (INT32_MAX) is returned as it is, unsafe
    False."""
    k = np.asarray(ss_time, np.int64)
    unsafe = (k >= LANE_UNSAFE_KEY) & (k != 0x7FFFFFFF)
    t = np.where(unsafe, k - LANE_UNSAFE_KEY, k)
    if t.ndim == 0:
        return int(t), bool(unsafe)
    return t.astype(np.int32), unsafe


# The (N, numSS_Points) pairs the library instantiates the QP kernel for: LMPC_FOR_EACH_CASE in csrc/ftocp_launch.cuh (a CPU test
# keeps the two equal)
SHAPE_GRID = tuple([(n, 0) for n in (4, 6, 8, 10, 12, 14, 16, 20, 24, 32, 48)] + [(n, 48) for n in (4, 6, 8, 10, 12, 14, 16, 20, 24, 32, 48)] +
                   [(n, m) for n in (12, 14) for m in (24, 32, 64, 96)])


class TrackParams(C.Structure):
    """lmpc_track_params: the [s_start, length, curvature] rows of Map.PointAndTangent and the lap length."""
    _fields_ = [("nseg", C.c_int), ("seg", C.c_double * (MAX_SEG * 3)), ("TrackLength", C.c_double)]


class LapReport(C.Structure):
    """lmpc_lap_report: one lap of one controller of the device closed loop (lmpc_rollout_enable_lap_reports)."""
    _fields_ = [("steps", C.c_int), ("flags", C.c_int), ("unsolved", C.c_int), ("viol_steps", C.c_int), ("ipm_iters", C.c_int),
                ("ipm_iters_max", C.c_int), ("viol_max", C.c_double)]


LAP_REPORT_FIELDS = tuple(f for f, _ in LapReport._fields_)
LAP_REPORT_DTYPE = np.dtype([(f, np.float64 if f == "viol_max" else np.int32) for f in LAP_REPORT_FIELDS])
MAX_LAP_REPORTS = 1024


def check_lap_reports(max_laps):
    """The capacity of BatchedController.enable_lap_reports: an integer 0 .. MAX_LAP_REPORTS (0 turns reports off).  Returns it as
    an int; raises ValueError."""
    if isinstance(max_laps, (bool, np.bool_)) or not isinstance(max_laps, (int, np.integer)):
        raise ValueError("max_laps must be an integer, got %r" % (max_laps,))
    if not 0 <= int(max_laps) <= MAX_LAP_REPORTS:
        raise ValueError("max_laps must be 0 .. %d, got %d" % (MAX_LAP_REPORTS, int(max_laps)))
    return int(max_laps)


SNAPSHOT_MAGIC, SNAPSHOT_VERSION, SNAPSHOT_SECTIONS = 0x50414E53, 1, 40
# the layout ints of a record header, in header order (lmpc_snapshot_header)
SNAPSHOT_LAYOUT = ("N", "M", "ncx", "ncu", "numSS_it", "trToUse", "ss_cap", "model_cap", "Tmax", "Tcl", "warm_start")
# section slots of a record, in header order (csrc/snapshot.cuh, SnapSection); DESIGN.md "Controller snapshots"
SNAPSHOT_SECTIONS_NAMES = ("ss_x", "ss_u", "ss_q", "ss_len", "model_x", "model_u", "model_len",
                           "ss_time", "ss_lap", "it", "md_time", "md_seq", "md_cnt", "lap_hist", "lap_n", "sel", "is_prev", "prev_slot",
                           "used", "xLin", "uLin", "zt", "OldInput", "xPredPrev", "timeStep", "has_pred", "warm", "warm_valid",
                           "x", "xglob", "cl_x", "cl_u", "cl_len", "done", "health_flags", "health_unsolved", "abc_lti",
                           "lap_reports", "lap_report_run")
# every section slot 0 .. 39: the slots above and the lane margins of lmpc_set_lane_margins in the last one
SNAPSHOT_SLOT_NAMES = SNAPSHOT_SECTIONS_NAMES + ("lane_margin",)


class SnapshotHeader(C.Structure):
    """lmpc_snapshot_header: the first bytes of every controller snapshot record."""
    _fields_ = ([("magic", C.c_int), ("version", C.c_int), ("bytes", C.c_int)] + [(f, C.c_int) for f in SNAPSHOT_LAYOUT] +
                [("warm_mode", C.c_int), ("nsect", C.c_int), ("sect_off", C.c_int * SNAPSHOT_SECTIONS),
                 ("sect_bytes", C.c_int * SNAPSHOT_SECTIONS), ("track", TrackParams)])


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
    L.lmpc_rollout_set_noise.argtypes = [_vp, C.POINTER(NoiseParams), C.c_int, _vp]
    L.lmpc_rollout_set_noise_streams.argtypes = [_vp, _vp]
    L.lmpc_rollout_set_measurement_noise.argtypes = [_vp, C.POINTER(MeasurementParams), C.c_int, _vp]
    L.lmpc_rollout_set_observers.argtypes = [_vp, C.POINTER(ObserverParams), C.c_int, _vp]
    L.lmpc_rollout_set_observer_priors.argtypes = [_vp, C.POINTER(ObserverPriorParams), C.c_int, _vp]
    L.lmpc_rollout_set_observer_gains.argtypes = [_vp, C.POINTER(ObserverGainParams), C.c_int, _vp]
    L.lmpc_rollout_set_lap_budget.argtypes = [_vp, _vp]
    L.lmpc_rollout_enable_lap_reports.argtypes = [_vp, C.c_int]
    L.lmpc_rollout_get_lap_reports.argtypes = [_vp, _vp, _vp]
    L.lmpc_rollout_set_lap_schedule.argtypes = [_vp, C.c_int, C.c_int, _vp]
    L.lmpc_set_tracks.argtypes = [_vp, C.POINTER(TrackParams), C.c_int, _vp]
    L.lmpc_set_regression_sets.argtypes = [_vp, C.POINTER(RegressionParams), C.c_int, _vp]
    L.lmpc_set_shapes.argtypes = [_vp, C.POINTER(ShapeParams), C.c_int, _vp]
    L.lmpc_set_ss_laps.argtypes = [_vp, C.POINTER(SsLapsParams), C.c_int, _vp]
    L.lmpc_set_lap_windows.argtypes = [_vp, C.POINTER(LapWindowParams), C.c_int, _vp]
    L.lmpc_set_lane_rules.argtypes = [_vp, C.POINTER(LaneRuleParams), C.c_int, _vp]
    L.lmpc_set_lane_margins.argtypes = [_vp, C.POINTER(LaneMarginParams), C.c_int, _vp]
    L.lmpc_get_lane_margins.argtypes = [_vp, _vp]
    L.lmpc_set_prediction_models.argtypes = [_vp, C.POINTER(PredictionModelParams), C.c_int, _vp]
    L.lmpc_rollout_set_surfaces.argtypes = [_vp, C.POINTER(SurfaceParams), C.c_int, _vp]
    L.lmpc_rollout_sysid.argtypes = [_vp, C.c_double, _vp, _vp]
    L.lmpc_rollout_seed_from_record.argtypes = [_vp, C.c_int, C.c_int, C.c_int]
    L.lmpc_rollout_get_lap.argtypes = [_vp, C.c_int, ip, _vp, _vp]
    L.lmpc_rollout_commit_laps.argtypes = [_vp, _vp, _vp, _vp]
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
    L.lmpc_rollout_group_stats.argtypes = [_vp, _vp]
    L.lmpc_pool_export_dev.argtypes = [_vp, C.c_int, C.c_int, C.c_longlong, _vp, _vp]
    L.lmpc_pool_export_groups_dev.argtypes = [_vp, C.c_int, C.c_int, C.c_longlong, _vp, _vp, _vp]
    L.lmpc_pool_import_dev.argtypes = [_vp, C.c_int, C.c_int, C.c_int, C.c_longlong, _vp, _vp, _vp]
    L.lmpc_set_pool_groups.argtypes = [_vp, C.c_int, _vp]
    L.lmpc_set_pool_min_overrun.argtypes = [_vp, C.c_int]
    L.lmpc_host_alloc.argtypes = [C.c_int, C.c_size_t, C.POINTER(_vp)]
    L.lmpc_host_free.argtypes = [_vp]
    L.lmpc_host_numa_node.argtypes = [C.c_int]
    L.lmpc_host_page_nodes.argtypes = [_vp, C.c_size_t, C.c_int, _vp]
    L.lmpc_sizeof_snapshot_header.restype = C.c_int
    L.lmpc_snapshot_bytes.argtypes = [_vp, C.POINTER(C.c_size_t)]
    L.lmpc_snapshot_pack_dev.argtypes = [_vp, C.c_int, _vp, _vp]
    L.lmpc_snapshot_unpack_dev.argtypes = [_vp, _vp, C.c_int, C.c_int, _vp, _vp]
    L.lmpc_rollout_get_clock.argtypes = [_vp, C.POINTER(C.c_ulonglong)]
    L.lmpc_rollout_set_clock.argtypes = [_vp, C.c_ulonglong]
    L.lmpc_sizeof_params.restype = C.c_int
    L.lmpc_sizeof_model_params.restype = C.c_int
    L.lmpc_sizeof_vehicle_params.restype = C.c_int
    L.lmpc_sizeof_track_params.restype = C.c_int
    L.lmpc_sizeof_noise_params.restype = C.c_int
    L.lmpc_sizeof_measurement_params.restype = C.c_int
    L.lmpc_sizeof_regression_params.restype = C.c_int
    L.lmpc_sizeof_shape_params.restype = C.c_int
    assert L.lmpc_sizeof_shape_params() == C.sizeof(ShapeParams), "lmpc_shape_params ABI mismatch"
    L.lmpc_sizeof_ss_laps_params.restype = C.c_int
    assert L.lmpc_sizeof_ss_laps_params() == C.sizeof(SsLapsParams), "lmpc_ss_laps_params ABI mismatch"
    L.lmpc_sizeof_lap_window_params.restype = C.c_int
    assert L.lmpc_sizeof_lap_window_params() == C.sizeof(LapWindowParams), "lmpc_lap_window_params ABI mismatch"
    L.lmpc_sizeof_lane_rule_params.restype = C.c_int
    assert L.lmpc_sizeof_lane_rule_params() == C.sizeof(LaneRuleParams), "lmpc_lane_rule_params ABI mismatch"
    L.lmpc_sizeof_lane_margin_params.restype = C.c_int
    assert L.lmpc_sizeof_lane_margin_params() == C.sizeof(LaneMarginParams), "lmpc_lane_margin_params ABI mismatch"
    L.lmpc_sizeof_prediction_model_params.restype = C.c_int
    assert L.lmpc_sizeof_prediction_model_params() == C.sizeof(PredictionModelParams), "lmpc_prediction_model_params ABI mismatch"
    L.lmpc_sizeof_surface_params.restype = C.c_int
    assert L.lmpc_sizeof_surface_params() == C.sizeof(SurfaceParams), "lmpc_surface_params ABI mismatch"
    L.lmpc_sizeof_lap_report.restype = C.c_int
    assert L.lmpc_sizeof_lap_report() == C.sizeof(LapReport), "lmpc_lap_report ABI mismatch"
    assert L.lmpc_sizeof_noise_params() == C.sizeof(NoiseParams), "lmpc_noise_params ABI mismatch"
    assert L.lmpc_sizeof_measurement_params() == C.sizeof(MeasurementParams), "lmpc_measurement_params ABI mismatch"
    L.lmpc_sizeof_observer_params.restype = C.c_int
    assert L.lmpc_sizeof_observer_params() == C.sizeof(ObserverParams), "lmpc_observer_params ABI mismatch"
    L.lmpc_sizeof_observer_prior_params.restype = C.c_int
    assert L.lmpc_sizeof_observer_prior_params() == C.sizeof(ObserverPriorParams), "lmpc_observer_prior_params ABI mismatch"
    L.lmpc_sizeof_observer_gain_params.restype = C.c_int
    assert L.lmpc_sizeof_observer_gain_params() == C.sizeof(ObserverGainParams), "lmpc_observer_gain_params ABI mismatch"
    assert L.lmpc_sizeof_regression_params() == C.sizeof(RegressionParams), "lmpc_regression_params ABI mismatch"
    assert L.lmpc_sizeof_params() == C.sizeof(Params), "lmpc_params ABI mismatch"
    assert L.lmpc_sizeof_model_params() == C.sizeof(ModelParams), "lmpc_model_params ABI mismatch"
    assert L.lmpc_sizeof_vehicle_params() == C.sizeof(VehicleParams), "lmpc_vehicle_params ABI mismatch"
    assert L.lmpc_sizeof_track_params() == C.sizeof(TrackParams), "lmpc_track_params ABI mismatch"
    assert L.lmpc_sizeof_snapshot_header() == C.sizeof(SnapshotHeader), "lmpc_snapshot_header ABI mismatch"
    _LIB = L
    return L


def make_model_params(seg_table, TrackLength, trToUse, MaxNumPoint=7, h=5.0, lamb=0.0, dt=0.1,
                      scaling=(0.1, 1.0, 1.0, 1.0, 1.0)):
    """PredictiveModel.__init__ constants (PredictiveModel.py:12-32) + the track's [s0, length, curvature] rows."""
    m = ModelParams()
    m.trToUse, m.MaxNumPoint = int(trToUse), int(MaxNumPoint)
    m.h, m.lamb, m.dt = float(h), float(lamb), float(dt)
    m.scaling[:] = list(scaling)
    _pack_track(m, seg_table, TrackLength)
    return m


def _pack_track(row, seg_table, TrackLength):
    """Writes a track into ``row`` (ModelParams or TrackParams): nseg, the [nseg, 3] segment rows zero-padded to MAX_SEG rows, and
    TrackLength.  Raises ValueError for more than MAX_SEG rows."""
    seg = np.asarray(seg_table, float).reshape(-1, 3)
    if seg.shape[0] > MAX_SEG:
        raise ValueError("track table has more than %d segments" % MAX_SEG)
    row.nseg = seg.shape[0]
    buf = np.zeros(MAX_SEG * 3)
    buf[:seg.size] = seg.ravel()
    row.seg[:] = buf
    row.TrackLength = float(TrackLength)


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
    """The index rules of the per-controller tables (lmpc_set_param_sets, lmpc_rollout_set_vehicles, lmpc_rollout_set_noise,
    lmpc_rollout_set_measurement_noise, lmpc_set_tracks, lmpc_set_regression_sets) and of the pool
    groups (lmpc_set_pool_groups): 1 <= K <= batch rows and
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


def _pack_sets(ctype, items, index, batch, what, make_row):
    """The rows and the index of a per-controller table: the index rules of ``_set_index`` for K = len(items) ``what``, then
    ``make_row(k, item)`` checks item k (raising ValueError) and returns its ``ctype`` row.  Returns (ctypes array ctype * K,
    int32 index array)."""
    items = list(items)
    idx = _set_index(index, len(items), batch, what)
    out = (ctype * len(items))()
    for k, item in enumerate(items):
        out[k] = make_row(k, item)
    return out, idx


def make_param_sets(base, params, index, batch, numSS_Points=0, numSS_it=0, QterminalSlack=None):
    """Per-controller parameters for ``lmpc_set_param_sets``: K MPCParams-like objects ``params``, the set of every controller
    ``index[batch]`` and ``QterminalSlack`` (None: the base's, or one 6x6 matrix per set).  ``base`` is the handle's own ``Params``;
    the interior-point settings (tolerances, max_iter, warm_start) are taken from it.  Each set is converted by ``make_params``.
    Raises ValueError where the library would refuse: an index of the wrong length or out of range, or a set that differs from
    the base in N, the rows of Fx or Fu, slacks or n/d.  Returns (ctypes array Params * K, int32 index array)."""
    params = list(params)
    if QterminalSlack is None:
        qts = [np.ctypeslib.as_array(base.QterminalSlack).reshape(6, 6).copy()] * len(params)
    else:
        qts = list(QterminalSlack)
        if len(qts) != len(params):
            raise ValueError("QterminalSlack needs one matrix per set (%d)" % len(params))

    def row(k, p):
        s = make_params(p, numSS_Points, numSS_it, qts[k], base.eps_res, base.eps_gap, base.max_iter, base.eps_step,
                        bool(base.warm_start))
        if (s.N, s.ncx, s.ncu) != (base.N, base.ncx, base.ncu):
            raise ValueError("set %d: N / rows of Fx / rows of Fu (%d, %d, %d) differ from the handle's (%d, %d, %d)"
                             % (k, s.N, s.ncx, s.ncu, base.N, base.ncx, base.ncu))
        if (s.numSS_Points, s.numSS_it) != (base.numSS_Points, base.numSS_it):
            raise ValueError("set %d: numSS_Points / numSS_it differ from the handle's" % k)
        return s
    return _pack_sets(Params, params, index, batch, "parameter sets", row)


VEHICLE_FIELDS = tuple(f for f, _ in VehicleParams._fields_)


def make_vehicle_sets(vehicles, index, batch):
    """Per-controller vehicles for ``lmpc_rollout_set_vehicles``: K objects ``vehicles`` with the reference's field names (m, lf,
    lr, Iz, Df, Cf, Bf, Dr, Cr, Br; e.g. reference_params.VehicleParams) and the vehicle of every controller ``index[batch]``.
    Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, a non-positive m, Iz, lf or lr,
    or a value that is not finite.  Returns (ctypes array VehicleParams * K, int32 index array)."""
    def row(k, v):
        vals = [float(getattr(v, f)) for f in VEHICLE_FIELDS]
        if not all(np.isfinite(vals)):
            raise ValueError("vehicle %d: every value must be finite" % k)
        if min(v.m, v.Iz, v.lf, v.lr) <= 0:
            raise ValueError("vehicle %d: m, Iz, lf and lr must be positive" % k)
        return VehicleParams(*vals)
    return _pack_sets(VehicleParams, vehicles, index, batch, "vehicles", row)


def make_surface_sets(surfaces, index, batch):
    """Per-controller track surfaces for ``lmpc_rollout_set_surfaces``: K objects ``surfaces`` with ``zones``, a sequence of
    (s_start, s_end, mu_f, mu_r) (e.g. reference_params.SurfaceParams), and the surface of every controller ``index[batch]``.
    Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, more than MAX_ZONES zones, a value
    that is not finite, s_start < 0, s_start >= s_end, a negative mu, or zones that do not ascend without overlap.  Returns
    (ctypes array SurfaceParams * K, int32 index array)."""
    def row(k, srf):
        zones = [tuple(float(v) for v in z) for z in srf.zones]
        if len(zones) > MAX_ZONES:
            raise ValueError("surface %d: at most %d zones, got %d" % (k, MAX_ZONES, len(zones)))
        r = SurfaceParams()
        r.nzone = len(zones)
        for j, z in enumerate(zones):
            if len(z) != 4:
                raise ValueError("surface %d, zone %d: a zone is (s_start, s_end, mu_f, mu_r)" % (k, j))
            s0, s1, muf, mur = z
            if not all(np.isfinite(z)):
                raise ValueError("surface %d, zone %d: s_start, s_end, mu_f and mu_r must be finite" % (k, j))
            if not 0.0 <= s0 < s1:
                raise ValueError("surface %d, zone %d: needs 0 <= s_start < s_end, got [%r, %r)" % (k, j, s0, s1))
            if muf < 0.0 or mur < 0.0:
                raise ValueError("surface %d, zone %d: mu_f and mu_r must be >= 0" % (k, j))
            if j and not zones[j - 1][1] <= s0:
                raise ValueError("surface %d, zone %d: zones must ascend without overlap (previous s_end %r > s_start %r)"
                                 % (k, j, zones[j - 1][1], s0))
            r.zone[4 * j:4 * j + 4] = list(z)
        return r
    return _pack_sets(SurfaceParams, surfaces, index, batch, "surfaces", row)


NOISE_FIELDS = tuple(f for f, _ in NoiseParams._fields_)


def make_noise_sets(noises, index, batch):
    """Per-controller noise models for ``lmpc_rollout_set_noise``: K objects ``noises`` with the fields of NoiseParams
    (sim_sigma[3], sim_clip[3], sim_gain, pid_sigma[2], pid_clip[2]; e.g. reference_params.NoiseParams) and the noise set of every
    controller ``index[batch]``.  Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, a
    field of the wrong length, or a value that is not finite or is negative.  Returns (ctypes array NoiseParams * K, int32 index
    array)."""
    def row(k, n):
        r = NoiseParams()
        for f, ct in NoiseParams._fields_:
            v = np.asarray(getattr(n, f), dtype=float).reshape(-1)
            want = getattr(ct, "_length_", 1)
            if v.shape[0] != want:
                raise ValueError("noise set %d: %s needs %d value%s, got %d" % (k, f, want, "s" if want > 1 else "", v.shape[0]))
            if not np.all(np.isfinite(v)) or np.any(v < 0):
                raise ValueError("noise set %d: %s must be finite and >= 0" % (k, f))
            if want > 1:
                getattr(r, f)[:] = v.tolist()
            else:
                setattr(r, f, float(v[0]))
        return r
    return _pack_sets(NoiseParams, noises, index, batch, "noise sets", row)


def make_measurement_sets(meas, index, batch):
    """Per-controller measurement noise for ``lmpc_rollout_set_measurement_noise``: K objects ``meas`` with the fields of
    MeasurementParams (sigma[6], clip[6] over vx, vy, wz, epsi, s, ey; e.g. reference_params.MeasurementParams) and the
    measurement set of every controller ``index[batch]``.  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets``, a field of the wrong length, or a value that is not finite or is negative.  Returns (ctypes array
    MeasurementParams * K, int32 index array)."""
    def row(k, m):
        r = MeasurementParams()
        for f, _ in MeasurementParams._fields_:
            v = np.asarray(getattr(m, f), dtype=float).reshape(-1)
            if v.shape[0] != 6:
                raise ValueError("measurement set %d: %s needs 6 values, got %d" % (k, f, v.shape[0]))
            if not np.all(np.isfinite(v)) or np.any(v < 0):
                raise ValueError("measurement set %d: %s must be finite and >= 0" % (k, f))
            getattr(r, f)[:] = v.tolist()
        return r
    return _pack_sets(MeasurementParams, meas, index, batch, "measurement sets", row)


def make_observer_sets(observers, index, batch):
    """Per-controller state observers for ``lmpc_rollout_set_observers``: K objects ``observers`` with ``mode`` (0 none, 1
    observer) and ``gain`` (six gains over vx, vy, wz, epsi, s, ey; e.g. reference_params.ObserverParams) and the observer of
    every controller ``index[batch]``.  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets``, a mode other than 0 or 1, a gain field of the wrong length, or a gain that is not finite or lies outside
    [0, 1].  Returns (ctypes array ObserverParams * K, int32 index array)."""
    def row(k, o):
        mode = o.mode
        if isinstance(mode, (bool, np.bool_)) or not isinstance(mode, (int, np.integer)) or int(mode) not in (0, 1):
            raise ValueError("observer %d: mode must be 0 or 1, got %r" % (k, mode))
        g = np.asarray(o.gain, dtype=float).reshape(-1)
        if g.shape[0] != 6:
            raise ValueError("observer %d: gain needs 6 values, got %d" % (k, g.shape[0]))
        if not np.all(np.isfinite(g)) or np.any(g < 0) or np.any(g > 1):
            raise ValueError("observer %d: every gain must be finite and in [0, 1]" % k)
        r = ObserverParams()
        r.mode = int(mode)
        r.gain[:] = g.tolist()
        return r
    return _pack_sets(ObserverParams, observers, index, batch, "observers", row)


def make_observer_gain_sets(gains, index, batch):
    """Per-controller observer gains for ``lmpc_rollout_set_observer_gains``: K objects ``gains`` with ``mode`` (0 the observer
    row's fixed gains, 1 model gains) and, read under mode 1, ``q`` and ``r`` (six values each over vx, vy, wz, epsi, s, ey; e.g.
    reference_params.ObserverGains), and the row of every controller ``index[batch]``.  Raises ValueError where the library would
    refuse a row: the index rules of ``make_param_sets``, a mode that is not the integer 0 or 1, or under mode 1 a q or r of the
    wrong length or with a value that is not finite and > 0.  (The library also refuses a mode 1 row for a controller without a
    source 1 or 2 observer prior; that needs the handle and is raised by its call.)  Returns (ctypes array ObserverGainParams *
    K, int32 index array)."""
    def row(k, o):
        mode = o.mode
        if isinstance(mode, (bool, np.bool_)) or not isinstance(mode, (int, np.integer)) or int(mode) not in (0, 1):
            raise ValueError("observer gains %d: mode must be 0 or 1, got %r" % (k, mode))
        r = ObserverGainParams()
        r.mode = int(mode)
        if r.mode == 0:
            return r
        for f in ("q", "r"):
            v = np.asarray(getattr(o, f), dtype=float).reshape(-1)
            if v.shape[0] != 6:
                raise ValueError("observer gains %d: %s needs 6 values, got %d" % (k, f, v.shape[0]))
            if not np.all(np.isfinite(v)) or np.any(v <= 0):
                raise ValueError("observer gains %d: every %s must be finite and > 0" % (k, f))
            getattr(r, f)[:] = v.tolist()
        return r
    return _pack_sets(ObserverGainParams, gains, index, batch, "observer gains", row)


def make_observer_prior_sets(priors, index, batch):
    """Per-controller observer priors for ``lmpc_rollout_set_observer_priors``: K objects ``priors`` with ``source`` (0 own plan,
    1 a believed car, 2 the plant's car) and ``vehicle`` (an object with the reference's ten vehicle field names, read under
    source 1; e.g. reference_params.ObserverPrior) and the row of every controller ``index[batch]``.  Raises ValueError where the
    library would refuse: the index rules of ``make_param_sets``, a source that is not the integer 0, 1 or 2, or a source 1
    vehicle with a value that is not finite or with m, lf, lr or Iz not positive.  Returns (ctypes array ObserverPriorParams * K,
    int32 index array)."""
    def row(k, r):
        src = r.source
        if isinstance(src, (bool, np.bool_)) or not isinstance(src, (int, np.integer)) or int(src) not in (0, 1, 2):
            raise ValueError("observer prior %d: source must be 0, 1 or 2, got %r" % (k, src))
        if int(src) != 1:
            return ObserverPriorParams(int(src), 0, VehicleParams())
        vals = []
        for f in VEHICLE_FIELDS:
            v = getattr(r.vehicle, f)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(float(v)):
                raise ValueError("observer prior %d: vehicle %s must be a finite number, got %r" % (k, f, v))
            vals.append(float(v))
        if min(vals[0], vals[1], vals[2], vals[3]) <= 0:
            raise ValueError("observer prior %d: a source 1 vehicle needs m, lf, lr and Iz > 0" % k)
        return ObserverPriorParams(1, 0, VehicleParams(*vals))
    return _pack_sets(ObserverPriorParams, priors, index, batch, "observer priors", row)


def _int_per_controller(values, batch, lo, what):
    """One integer >= lo per controller ``values[batch]`` as a contiguous int32 array (the arrays without a table:
    lmpc_rollout_set_noise_streams, lmpc_rollout_set_lap_budget); raises ValueError."""
    s = np.asarray(values).reshape(-1)
    with np.errstate(invalid="ignore"):              # NaN or an out-of-range value fails the comparison below
        out = np.ascontiguousarray(s, dtype=np.int32)
    if out.shape[0] != batch or not np.array_equal(out, s):
        raise ValueError("need one integer %s per controller (%d)" % (what, batch))
    if out.min() < lo:
        raise ValueError("every %s must be >= %d" % (what, lo))
    return out


def make_noise_streams(streams, batch):
    """Noise streams for ``lmpc_rollout_set_noise_streams``: one integer stream number >= 0 per controller ``streams[batch]``
    (repeats allowed: controllers on one stream meet the same Philox draws).  ``None`` (stream b = b) returns None.  Raises
    ValueError where the library would refuse.  Returns the int32 stream array."""
    return None if streams is None else _int_per_controller(streams, batch, 0, "stream number")


def make_lap_budget(budget, batch):
    """Lap budgets for ``lmpc_rollout_set_lap_budget``: the laps every controller drives before it retires, one integer >= 1 for
    the whole batch or one per controller ``budget[batch]``.  ``None`` (no budget) returns None.  Raises ValueError where the
    library would refuse.  Returns the int32 budget array."""
    if budget is None:
        return None
    if np.ndim(budget) == 0:
        budget = [budget] * batch
    return _int_per_controller(budget, batch, 1, "lap budget")


# lmpc_rollout_set_lap_schedule: the tables a lap schedule can index (LMPC_SCHEDULE_*) and the longest schedule
LAP_SCHEDULE_TABLES = {"vehicle": 0, "noise": 1, "measurement": 2, "surface": 3}
MAX_LAP_SCHEDULE = 1024


def make_lap_schedule(rows, batch, nsets):
    """A lap schedule for ``lmpc_rollout_set_lap_schedule``: the row of a table of ``nsets`` rows that every controller drives each
    LMPC lap under, ``rows[L]`` (the same for every controller) or ``rows[batch, L]``, 1 <= L <= 1024; the last entry holds for
    every later lap.  Raises ValueError where the library would refuse: another shape, entries that are not integers, L outside
    1 .. 1024, or an entry outside [0, nsets).  Returns the [batch, L] schedule as a contiguous int32 array."""
    a = np.asarray(rows)
    if a.ndim not in (1, 2) or a.size == 0:
        raise ValueError("a lap schedule is [L] or [batch, L] with L >= 1, got shape %s" % (a.shape,))
    if a.dtype.kind not in "iu" and not (a.dtype.kind == "f" and np.all(np.isfinite(a)) and np.array_equal(a, np.round(a))):
        raise ValueError("lap schedule entries must be integer row numbers")
    if a.ndim == 2 and a.shape[0] != int(batch):
        raise ValueError("a [batch, L] lap schedule needs %d rows, got %d" % (int(batch), a.shape[0]))
    L = a.shape[-1]
    if not 1 <= L <= MAX_LAP_SCHEDULE:
        raise ValueError("a lap schedule holds 1 .. %d laps, got %d" % (MAX_LAP_SCHEDULE, L))
    if a.min() < 0 or a.max() >= int(nsets):
        raise ValueError("lap schedule entry out of range [0, %d): the table has %d row(s)" % (int(nsets), int(nsets)))
    return np.ascontiguousarray(np.broadcast_to(a, (int(batch), L)), dtype=np.int32)


# the scaling entries the regression sets admit: 0 or this range (the fp32 pre-filter of K1 is certified there, csrc/safeset.cuh)
SCALING_MIN, SCALING_MAX = 2.0 ** -32, 2.0 ** 32
H_MIN, H_MAX = 2.0 ** -1022, 2.0 ** 1022


def make_regression_sets(regs, index, batch, trToUse):
    """Per-controller regression models for ``lmpc_set_regression_sets``: K objects ``regs`` with the fields of RegressionParams
    (trToUse, MaxNumPoint, h, lamb, scaling[5]; e.g. reference_params.RegressionParams) and the regression set of every
    controller ``index[batch]``; ``trToUse`` is the store's.  Raises ValueError where the library would refuse: the index rules
    of ``make_param_sets``, 1 <= trToUse <= the store's, 1 <= MaxNumPoint <= 7, h finite in [2^-1022, 2^1022], lamb finite and
    >= 0, five finite scaling entries with |s| == 0 or 2^-32 <= |s| <= 2^32.  Returns (ctypes array RegressionParams * K, int32
    index array); the scaling is packed as given (the library takes |s|)."""
    def row(k, r):
        w = "regression set %d: " % k
        for f in ("trToUse", "MaxNumPoint"):
            v = getattr(r, f)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
                raise ValueError(w + "%s must be an integer" % f)
        if not 1 <= int(r.trToUse) <= int(trToUse):
            raise ValueError(w + "trToUse must be 1 .. the store's trToUse (%d), got %d" % (trToUse, r.trToUse))
        if not 1 <= int(r.MaxNumPoint) <= 7:
            raise ValueError(w + "MaxNumPoint must be 1 .. 7, got %d" % r.MaxNumPoint)
        h, lamb = float(r.h), float(r.lamb)
        if not H_MIN <= h <= H_MAX:
            raise ValueError(w + "h must be finite and in [2^-1022, 2^1022], got %r" % h)
        if not (np.isfinite(lamb) and lamb >= 0):
            raise ValueError(w + "lamb must be finite and >= 0, got %r" % lamb)
        s = np.asarray(r.scaling, dtype=float).reshape(-1)
        if s.shape[0] != 5:
            raise ValueError(w + "scaling needs 5 values, got %d" % s.shape[0])
        a = np.abs(s)
        if not np.all(np.isfinite(s)) or not np.all((a == 0) | ((a >= SCALING_MIN) & (a <= SCALING_MAX))):
            raise ValueError(w + "every |scaling| must be 0 or in [2^-32, 2^32]")
        return RegressionParams(int(r.trToUse), int(r.MaxNumPoint), h, lamb, tuple(s.tolist()))
    return _pack_sets(RegressionParams, regs, index, batch, "regression sets", row)


def _even_split(M, nit):
    """M safe-set points split into nit laps of an even number of points each (PC.py:403,492-495)"""
    return M % nit == 0 and (M // nit) % 2 == 0


def make_shape_sets(shapes, index, batch, N, M, numSS_it, ss_laps=None):
    """Per-controller shapes for ``lmpc_set_shapes``: K ``(N, numSS_Points)`` pairs ``shapes`` and the shape of every controller
    ``index[batch]`` on a handle of horizon ``N``, safe-set size ``M`` and ``numSS_it`` laps.  Raises ValueError where the library
    would refuse: the index rules of ``make_param_sets``, a pair outside SHAPE_GRID, N or numSS_Points above the handle's, a
    numSS_Points that is 0 on an LMPC handle or > 0 on an MPC handle, or one that is not numSS_it times an even number of points
    per lap.  ``ss_laps`` (the numSS_it of every controller under ``lmpc_set_ss_laps``, or None) replaces numSS_it in that last
    check, controller by controller.  Returns (ctypes array ShapeParams * K, int32 index array)."""
    def row(k, sh):
        w = "shape %d: " % k
        try:
            n, m = sh
        except (TypeError, ValueError):
            raise ValueError(w + "need an (N, numSS_Points) pair, got %r" % (sh,))
        for v in (n, m):
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
                raise ValueError(w + "N and numSS_Points must be integers, got %r" % (sh,))
        n, m = int(n), int(m)
        if (n, m) not in SHAPE_GRID:
            raise ValueError(w + "(%d, %d) is not an instantiated (N, numSS_Points) pair" % (n, m))
        if n > int(N) or m > int(M):
            raise ValueError(w + "(%d, %d) exceeds the handle's (%d, %d)" % (n, m, N, M))
        if (m > 0) != (int(M) > 0):
            raise ValueError(w + "numSS_Points must be > 0 exactly when the handle's is (%d)" % M)
        if ss_laps is None and m > 0 and not _even_split(m, int(numSS_it)):
            raise ValueError(w + "numSS_Points must be numSS_it (%d) times an even number of points per lap" % numSS_it)
        return ShapeParams(n, m)
    rows, idx = _pack_sets(ShapeParams, shapes, index, batch, "shapes", row)
    if ss_laps is not None:
        for b in range(batch):
            m, v = rows[idx[b]].numSS_Points, int(ss_laps[b])
            if not _even_split(m, v):
                raise ValueError("controller %d: numSS_Points %d is not its numSS_it (%d) times an even number of points per lap" % (b, m, v))
    return rows, idx


def make_ss_laps_sets(values, index, batch, numSS_it, points):
    """Per-controller safe-set lap counts for ``lmpc_set_ss_laps``: K values of numSS_it ``values`` and the value of every
    controller ``index[batch]`` on an LMPC handle of ``numSS_it`` laps whose controllers have ``points[batch]`` safe-set points
    (their shapes, or the handle's numSS_Points).  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets``, a value that is not an integer in 1 .. numSS_it, or a controller whose points are not its value times an
    even number of points per lap.  Returns (ctypes array SsLapsParams * K, int32 index array)."""
    if int(numSS_it) < 1 or min(int(m) for m in points) <= 0:
        raise ValueError("per-controller lap counts need an LMPC handle (numSS_Points > 0)")

    def row(k, v):
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
            raise ValueError("lap count %d: numSS_it must be an integer, got %r" % (k, v))
        if not 1 <= int(v) <= int(numSS_it):
            raise ValueError("lap count %d: numSS_it must be 1 .. the handle's %d, got %d" % (k, numSS_it, v))
        return SsLapsParams(int(v))
    rows, idx = _pack_sets(SsLapsParams, values, index, batch, "lap counts", row)
    for b in range(batch):
        m, v = int(points[b]), rows[idx[b]].numSS_it
        if not _even_split(m, v):
            raise ValueError("controller %d: numSS_Points %d is not numSS_it (%d) times an even number of points per lap" % (b, m, v))
    return rows, idx


def make_lap_window_sets(windows, index, batch, ss_laps, ss_cap, trToUse, model_cap, lmpc=True):
    """Per-controller lap windows for ``lmpc_set_lap_windows``: K objects ``windows`` with ``ss_window`` and ``model_window``
    (e.g. reference_params.LapWindowParams; 0 = unbounded) and the row of every controller ``index[batch]``, on a store of
    ``ss_cap`` / ``model_cap`` slots and ``trToUse`` laps whose controllers have the lap counts ``ss_laps[batch]`` (their values
    under ``lmpc_set_ss_laps``, or the handle's numSS_it).  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets``, a window that is not an integer, an ss_window > 0 without a safe set (``lmpc`` False) or outside
    numSS_it_b .. ss_cap of a controller b of its row, a model_window outside trToUse .. model_cap.  Returns (ctypes array
    LapWindowParams * K, int32 index array)."""
    def row(k, w):
        vals = []
        for f in ("ss_window", "model_window"):
            v = getattr(w, f)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
                raise ValueError("lap window %d: %s must be an integer, got %r" % (k, f, v))
            vals.append(int(v))
        sw, mw = vals
        if sw != 0 and not lmpc:
            raise ValueError("lap window %d: ss_window must be 0: the handle has no safe set (numSS_Points == 0)" % k)
        if not (sw == 0 or 1 <= sw <= int(ss_cap)):
            raise ValueError("lap window %d: ss_window must be 0 or numSS_it .. ss_cap (%d), got %d" % (k, ss_cap, sw))
        if not (mw == 0 or int(trToUse) <= mw <= int(model_cap)):
            raise ValueError("lap window %d: model_window must be 0 or trToUse (%d) .. model_cap (%d), got %d" % (k, trToUse, model_cap, mw))
        return LapWindowParams(sw, mw)
    rows, idx = _pack_sets(LapWindowParams, windows, index, batch, "lap windows", row)
    for b in range(batch):
        w, v = rows[idx[b]].ss_window, int(ss_laps[b])
        if 0 < w < v:
            raise ValueError("controller %d: ss_window %d is below its numSS_it (%d)" % (b, w, v))
    return rows, idx


def make_lane_rule_sets(rules, index, batch, lmpc=True, Tcl=0):
    """Per-controller lane rules for ``lmpc_set_lane_rules``: K objects ``rules`` with ``mode`` (0 or 1) and ``lane_tol`` (e.g.
    reference_params.LaneRuleParams) and the row of every controller ``index[batch]``.  Raises ValueError where the library would
    refuse a value: the index rules of ``make_param_sets``, a handle without a safe set (``lmpc`` False), a mode that is not the
    integer 0 or 1, a lane_tol that is not a finite number >= 0, or a mode 1 row with a rollout of ``Tcl`` >= LANE_UNSAFE_KEY.
    Returns (ctypes array LaneRuleParams * K, int32 index array)."""
    if not lmpc:
        raise ValueError("lane rules need a safe set: the handle has numSS_Points == 0")

    def row(k, r):
        m, tol = r.mode, r.lane_tol
        if isinstance(m, (bool, np.bool_)) or not isinstance(m, (int, np.integer)) or int(m) not in (0, 1):
            raise ValueError("lane rule %d: mode must be 0 or 1, got %r" % (k, m))
        if isinstance(tol, (bool, np.bool_)) or not isinstance(tol, (int, float, np.integer, np.floating)):
            raise ValueError("lane rule %d: lane_tol must be a number, got %r" % (k, tol))
        if not (np.isfinite(float(tol)) and float(tol) >= 0.0):
            raise ValueError("lane rule %d: lane_tol must be finite and >= 0, got %r" % (k, tol))
        if int(m) == 1 and int(Tcl) >= LANE_UNSAFE_KEY:
            raise ValueError("lane rule %d: the rollout's Tcl (%d) must stay below LANE_UNSAFE_KEY" % (k, int(Tcl)))
        return LaneRuleParams(int(m), 0, float(tol))
    return _pack_sets(LaneRuleParams, rules, index, batch, "lane rules", row)


def make_lane_margin_sets(margins, index, batch, bx_min):
    """Per-controller lane margins for ``lmpc_set_lane_margins``: K objects ``margins`` with ``mode`` (0, 1 or 2), ``margin0``,
    ``margin_max``, ``step_up`` and ``step_down`` (e.g. reference_params.LaneMarginParams) and the row of every controller
    ``index[batch]``; ``bx_min[batch]`` is min_i bx_i of the QP row each controller reads.  Raises ValueError where the library
    would refuse: the index rules of ``make_param_sets``, a mode that is not the integer 0, 1 or 2, a value that is not a finite
    number >= 0, margin0 > margin_max, or a margin that does not leave a lane (``check_margins_leave_lane``).  Returns (ctypes
    array LaneMarginParams * K, int32 index array)."""
    def row(k, r):
        m = r.mode
        if isinstance(m, (bool, np.bool_)) or not isinstance(m, (int, np.integer)) or int(m) not in (0, 1, 2):
            raise ValueError("lane margin %d: mode must be 0, 1 or 2, got %r" % (k, m))
        vals = []
        for f in ("margin0", "margin_max", "step_up", "step_down"):
            v = getattr(r, f)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)):
                raise ValueError("lane margin %d: %s must be a number, got %r" % (k, f, v))
            if not (np.isfinite(float(v)) and float(v) >= 0.0):
                raise ValueError("lane margin %d: %s must be finite and >= 0, got %r" % (k, f, v))
            vals.append(float(v))
        if vals[0] > vals[1]:
            raise ValueError("lane margin %d: margin0 (%r) must not exceed margin_max (%r)" % (k, vals[0], vals[1]))
        return LaneMarginParams(int(m), 0, *vals)
    rows, idx = _pack_sets(LaneMarginParams, margins, index, batch, "lane margins", row)
    check_margins_leave_lane(rows, idx, bx_min)
    return rows, idx


def make_prediction_model_sets(models, index, batch):
    """Per-controller prediction models for ``lmpc_set_prediction_models``: K objects ``models`` with ``mode`` (0, 1 or 2) and
    ``vehicle`` (an object with the reference's ten vehicle field names; e.g. reference_params.PredictionModelParams) and the row
    of every controller ``index[batch]``.  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets``, a mode that is not the integer 0, 1 or 2, a vehicle value that is not finite, or a mode 1 vehicle with
    m, lf, lr or Iz not positive.  Returns (ctypes array PredictionModelParams * K, int32 index array)."""
    def row(k, r):
        m = r.mode
        if isinstance(m, (bool, np.bool_)) or not isinstance(m, (int, np.integer)) or int(m) not in (0, 1, 2):
            raise ValueError("prediction model %d: mode must be 0, 1 or 2, got %r" % (k, m))
        vals = []
        for f in VEHICLE_FIELDS:
            v = getattr(r.vehicle, f)
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or not np.isfinite(float(v)):
                raise ValueError("prediction model %d: vehicle %s must be a finite number, got %r" % (k, f, v))
            vals.append(float(v))
        if int(m) == 1 and min(vals[0], vals[1], vals[2], vals[3]) <= 0:
            raise ValueError("prediction model %d: a mode 1 vehicle needs m, lf, lr and Iz > 0" % k)
        return PredictionModelParams(int(m), 0, VehicleParams(*vals))
    return _pack_sets(PredictionModelParams, models, index, batch, "prediction models", row)


def margin_width(r):
    """The widest margin a lane-margin row plans with: margin0 under mode 1, margin_max under mode 2, None under mode 0."""
    return None if int(r.mode) == 0 else float(r.margin0 if int(r.mode) == 1 else r.margin_max)


def check_margins_leave_lane(rows, idx, bx_min):
    """ValueError unless every controller's margin leaves a lane: margin_width(rows[idx[b]]) < bx_min[b] (min_i bx_i of the QP row
    controller b reads) wherever the row has a margin."""
    bx_min = np.asarray(bx_min, np.float64).reshape(-1)
    for k, r in enumerate(rows):
        w = margin_width(r)
        sel = np.nonzero(np.asarray(idx) == k)[0]
        if w is not None and sel.size and not (w < bx_min[sel]).all():
            b = int(sel[np.argmin(bx_min[sel])])
            raise ValueError("lane margin %d: the margin %r of controller %d does not leave a lane (its bx reaches %r)"
                             % (k, w, b, float(bx_min[b])))


def make_pool_groups(index, ngroups, batch):
    """Pool groups for ``lmpc_set_pool_groups``: the group of every controller ``index[batch]`` among ``ngroups``.  ``ngroups == 0``
    goes with ``index=None`` (one pool) and returns None.  Raises ValueError where the library would refuse: the index rules of
    ``make_param_sets`` (with groups for sets; a group may be empty), more than MAX_POOL_GROUPS groups, or an index with
    ``ngroups == 0``.  Returns the int32 index array."""
    ngroups = int(ngroups)
    if ngroups == 0:
        if index is not None:
            raise ValueError("ngroups == 0 returns to one pool and takes no index")
        return None
    if ngroups > MAX_POOL_GROUPS:
        raise ValueError("at most %d pool groups, got %d" % (MAX_POOL_GROUPS, ngroups))
    return _set_index(index, ngroups, batch, "pool groups")


def make_track_sets(tracks, index, batch):
    """Per-controller tracks for ``lmpc_set_tracks``: K objects ``tracks`` with ``seg_table`` ([nseg, 3] rows s_start, length,
    curvature) and ``TrackLength`` (e.g. reference_params.TrackParams) and the track of every controller ``index[batch]``.
    Raises ValueError where the library would refuse: the index rules of ``make_param_sets``, 1 .. 16 rows, a value that is not
    finite, a negative length, a first start other than 0, a start other than the previous start + length, or a TrackLength that
    is not positive or not the last start + length (all exact: Track.py:54-133 builds the table that way).
    Returns (ctypes array TrackParams * K, int32 index array)."""
    def row(k, t):
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
        r = TrackParams()
        _pack_track(r, seg, L)
        return r
    return _pack_sets(TrackParams, tracks, index, batch, "tracks", row)


# ---- controller snapshots: the checks the library makes, in Python, before any device work -----------------------------------
def decode_snapshot_header(raw):
    """Header of one snapshot record (bytes, or a uint8 array / CPU tensor holding at least the header) -> dict with magic, version,
    bytes, the layout ints (SNAPSHOT_LAYOUT), warm_mode, the sections {name: (offset, bytes)} present, and the track row
    (nseg, seg [nseg, 3], TrackLength).  Raises ValueError on a short buffer, a wrong magic or an unknown version."""
    buf = bytes(np.asarray(raw, dtype=np.uint8).reshape(-1)[:C.sizeof(SnapshotHeader)]) if not isinstance(raw, (bytes, bytearray)) \
        else bytes(raw[:C.sizeof(SnapshotHeader)])
    if len(buf) < C.sizeof(SnapshotHeader):
        raise ValueError("a snapshot record starts with a %d-byte header, got %d bytes" % (C.sizeof(SnapshotHeader), len(buf)))
    h = SnapshotHeader.from_buffer_copy(buf)
    if h.magic & 0xFFFFFFFF != SNAPSHOT_MAGIC:
        raise ValueError("not a controller snapshot record (magic 0x%08x)" % (h.magic & 0xFFFFFFFF))
    if h.version != SNAPSHOT_VERSION:
        raise ValueError("snapshot record version %d; this build reads version %d" % (h.version, SNAPSHOT_VERSION))
    out = {"magic": h.magic, "version": h.version, "bytes": h.bytes, "warm_mode": h.warm_mode}
    out.update({f: getattr(h, f) for f in SNAPSHOT_LAYOUT})
    out["sections"] = {n: (h.sect_off[k], h.sect_bytes[k]) for k, n in enumerate(SNAPSHOT_SLOT_NAMES) if h.sect_bytes[k] > 0}
    nseg = int(h.track.nseg)
    out["track"] = {"nseg": nseg, "seg": np.array(h.track.seg[:3 * max(0, min(nseg, MAX_SEG))]).reshape(-1, 3),
                    "TrackLength": float(h.track.TrackLength)}
    return out


def snapshot_lap_reports(header):
    """Report capacity L of a decoded header's record: 0 without report sections."""
    return header["sections"].get("lap_reports", (0, 0))[1] // C.sizeof(LapReport)


def snapshot_layout_mismatch(header, layout):
    """The first layout field in which a decoded header differs from ``layout`` (a dict with SNAPSHOT_LAYOUT keys and "bytes",
    "lap_reports" = the report capacity when reports are on and "lane_margin" = 1 under a lane-margin table), as a message, or None
    when the record fits.  The report capacity and the lane margin are compared before the size, which they change."""
    had, mine = snapshot_lap_reports(header), int(layout.get("lap_reports", 0))
    if had != mine:
        what = lambda L: "%d report rows" % L if L else "no lap reports"
        return "snapshot layout mismatch: lap_reports: the record has %s and this controller %s" % (what(had), what(mine))
    had, mine = int("lane_margin" in header["sections"]), int(layout.get("lane_margin", 0))
    if had != mine:
        what = lambda m: "a lane margin" if m else "no lane margin"
        return "snapshot layout mismatch: lane margin layout: the record has %s and this controller %s" % (what(had), what(mine))
    for f in SNAPSHOT_LAYOUT + ("bytes",):
        if int(header[f]) != int(layout[f]):
            return "snapshot layout mismatch: %s is %d in the record and %d in this controller" % (f, header[f], layout[f])
    return None


def snapshot_indices(index, batch, what, unique=False):
    """Controller indices of a snapshot call: None stays None (every controller), else a non-empty 1-D list of integers in
    [0, batch), unique when ``unique``.  Returns an int32 array; raises ValueError."""
    if index is None:
        return None
    a = np.asarray(index).reshape(-1)
    if a.size == 0:
        raise ValueError("%s: at least one controller" % what)
    idx = np.ascontiguousarray(a, dtype=np.int32)
    if not np.issubdtype(a.dtype, np.integer) or not np.array_equal(idx, a):
        raise ValueError("%s must hold integer controller indices" % what)
    if idx.min() < 0 or idx.max() >= batch:
        raise ValueError("%s: controller index out of range [0, %d)" % (what, batch))
    if unique and np.unique(idx).size != idx.size:
        raise ValueError("%s: a controller may be restored only once per call" % what)
    return idx


def snapshot_record_map(rec_of, n, nrec):
    """Record of every destination for an unpack: None = record i for destination i (needs nrec >= n), else n integers in
    [0, nrec).  Returns an int32 array; raises ValueError."""
    if rec_of is None:
        if nrec < n:
            raise ValueError("%d destinations and %d records: pass rec_of to map records onto destinations" % (n, nrec))
        return np.arange(n, dtype=np.int32)
    a = np.asarray(rec_of).reshape(-1)
    idx = np.ascontiguousarray(a, dtype=np.int32)
    if a.size != n or not np.issubdtype(a.dtype, np.integer) or not np.array_equal(idx, a):
        raise ValueError("rec_of needs one integer record index per destination (%d)" % n)
    if n and (idx.min() < 0 or idx.max() >= nrec):
        raise ValueError("rec_of: record index out of range [0, %d)" % nrec)
    return idx


def check_snapshot_tensor(t, device, nbytes, rows=None, what="records"):
    """A record buffer: a contiguous uint8 CUDA tensor [rows, nbytes] on cuda:``device`` whose data is 16-byte aligned.  Raises
    ValueError."""
    if not hasattr(t, "is_cuda") or not hasattr(t, "dtype"):
        raise ValueError("%s must be a torch tensor" % what)
    if str(t.dtype) != "torch.uint8":
        raise ValueError("%s must be uint8, got %s" % (what, t.dtype))
    if not t.is_cuda or t.device.index != int(device):
        raise ValueError("%s must live on cuda:%d, got %s" % (what, int(device), t.device))
    if t.dim() != 2 or t.shape[1] != nbytes or (rows is not None and t.shape[0] != rows) or t.shape[0] < 1:
        raise ValueError("%s must have shape [%s, %d], got %s" % (what, "n" if rows is None else rows, nbytes, tuple(t.shape)))
    if not t.is_contiguous() or t.data_ptr() % 16:
        raise ValueError("%s must be contiguous and 16-byte aligned" % what)
