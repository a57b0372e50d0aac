"""ctypes binding of the graph builder of libdynoba (include/dynoba.h, dynoba_builder_*): frames + observations in,
flat SoA problem out (SURVEY.md 8f-3; reference: Formulation-impl.hpp:552-897, HybridEstimator.cc:573-830)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .binding import DynobaError, OK, c_dp, c_ip, c_u64p, load
from .problem import ARITY, MEAS_DIM, FactorBlock, Problem

c_i64p = C.POINTER(C.c_int64)


class BuilderParams(C.Structure):
    _fields_ = [("min_static_obs", C.c_int32), ("min_dynamic_obs", C.c_int32), ("keyframe_gap", C.c_int32),
                ("sigma_static", C.c_double), ("sigma_dynamic", C.c_double), ("huber_k", C.c_double),
                ("odometry_sigma", C.c_double*6), ("smoothing_sigma", C.c_double*6), ("prior_sigma", C.c_double),
                ("formulation", C.c_int32), ("sigma_motion", C.c_double), ("backtrack", C.c_int32)]

FORMULATIONS = {"hybrid": 0, "wcme": 1, "wcpe": 2}


def _dp(a):
    return a.ctypes.data_as(c_dp)


class GraphBuilder:
    def __init__(self, **params):
        self.lib = load()
        L = self.lib
        L.dynoba_builder_last_error.restype = C.c_char_p
        L.dynoba_builder_last_error.argtypes = [C.c_void_p]
        L.dynoba_builder_create.argtypes = [C.POINTER(BuilderParams), C.POINTER(C.c_void_p)]
        L.dynoba_builder_add_frame.argtypes = [C.c_void_p, C.c_int32, c_dp, c_dp]
        L.dynoba_builder_add_static.argtypes = [C.c_void_p, C.c_int32, C.c_int64, c_i64p, c_dp]
        L.dynoba_builder_add_dynamic.argtypes = [C.c_void_p, C.c_int32, C.c_int64, c_i64p, c_ip, c_dp]
        L.dynoba_builder_set_motion_init.argtypes = [C.c_void_p, C.c_int32, C.c_int32, c_dp]
        L.dynoba_builder_set_keyframe_pose.argtypes = [C.c_void_p, C.c_int32, C.c_int32, c_dp]
        L.dynoba_builder_finalize.argtypes = [C.c_void_p]
        L.dynoba_builder_destroy.argtypes = [C.c_void_p]
        L.dynoba_builder_counts.argtypes = [C.c_void_p, c_i64p, c_i64p, c_i64p, C.POINTER(C.c_int32)]
        L.dynoba_builder_get_variables.argtypes = [C.c_void_p, c_dp, c_dp, c_dp, c_ip, c_u64p, c_u64p]
        L.dynoba_builder_block_info.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), c_i64p, C.POINTER(C.c_int32), c_i64p, c_dp, C.POINTER(C.c_int32)]
        L.dynoba_builder_get_block.argtypes = [C.c_void_p, C.c_int32, c_ip, c_dp, c_dp, c_ip]
        L.dynoba_builder_emit.argtypes = [C.c_void_p, C.c_void_p]
        L.dynoba_builder_set_imu.argtypes = [C.c_void_p, C.c_int32, c_dp, c_dp]
        L.dynoba_builder_nav_counts.argtypes = [C.c_void_p, c_i64p, c_i64p]
        L.dynoba_builder_get_nav_variables.argtypes = [C.c_void_p, c_dp, c_dp, c_ip, c_ip, c_u64p, c_u64p]
        L.dynoba_builder_set_static_stereo.argtypes = [C.c_void_p, c_dp, C.c_double, C.c_int]
        L.dynoba_builder_add_static_stereo.argtypes = [C.c_void_p, C.c_int32, C.c_int64, c_i64p, c_dp]
        L.dynoba_builder_static_stereo_stats.argtypes = [C.c_void_p, c_i64p, c_i64p, c_i64p]
        self.calib = None
        prm = BuilderParams(); L.dynoba_builder_default_params(C.byref(prm))
        for k, v in params.items():
            if k in ("odometry_sigma", "smoothing_sigma"):
                for i in range(6):
                    getattr(prm, k)[i] = float(v[i])
            elif k == "formulation":
                prm.formulation = FORMULATIONS[v] if isinstance(v, str) else int(v)
            else:
                setattr(prm, k, v)
        self.h = C.c_void_p()
        self._ck(L.dynoba_builder_create(C.byref(prm), C.byref(self.h)))

    def _ck(self, st):
        if st != OK:
            raise DynobaError(st, self.lib.dynoba_builder_last_error(self.h).decode() if self.h else "builder")

    def close(self):
        if self.h:
            self.lib.dynoba_builder_destroy(self.h); self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_frame(self, frame, X, odom_from_prev=None):
        X = np.ascontiguousarray(X, np.float64).reshape(12)
        od = None if odom_from_prev is None else np.ascontiguousarray(odom_from_prev, np.float64).reshape(12)
        self._ck(self.lib.dynoba_builder_add_frame(self.h, int(frame), _dp(X), _dp(od) if od is not None else C.cast(None, c_dp)))

    def add_static(self, frame, tracklet, z):
        t = np.ascontiguousarray(tracklet, np.int64); z = np.ascontiguousarray(z, np.float64).reshape(-1, 3)
        self._ck(self.lib.dynoba_builder_add_static(self.h, int(frame), t.size, t.ctypes.data_as(c_i64p), _dp(z)))

    def add_dynamic(self, frame, tracklet, obj, z):
        t = np.ascontiguousarray(tracklet, np.int64); o = np.ascontiguousarray(obj, np.int32); z = np.ascontiguousarray(z, np.float64).reshape(-1, 3)
        self._ck(self.lib.dynoba_builder_add_dynamic(self.h, int(frame), t.size, t.ctypes.data_as(c_i64p), o.ctypes.data_as(c_ip), _dp(z)))

    def set_motion_init(self, obj, frame, H):
        H = np.ascontiguousarray(H, np.float64).reshape(12); self._ck(self.lib.dynoba_builder_set_motion_init(self.h, int(obj), int(frame), _dp(H)))

    def set_keyframe_pose(self, obj, keyframe, L_e):
        L_e = np.ascontiguousarray(L_e, np.float64).reshape(12); self._ck(self.lib.dynoba_builder_set_keyframe_pose(self.h, int(obj), int(keyframe), _dp(L_e)))

    def set_imu(self, frame, record, sqrt_info):
        """the preintegrated measurement from the previous frame to `frame`: record[70] (COMBINED_IMU15 layout) and R[15, 15]"""
        z = np.ascontiguousarray(record, np.float64).reshape(70); R = np.ascontiguousarray(sqrt_info, np.float64).reshape(225)
        self._ck(self.lib.dynoba_builder_set_imu(self.h, int(frame), _dp(z), _dp(R)))

    def set_static_stereo(self, calib6, sigma_px, device=-1):
        """static landmarks by stereo projection (STEREO_PROJECTION): calib6 = fx fy s u0 v0 baseline, sigma_px the pixel sigma
        of the GenericStereoFactors, device the GPU that triangulates at finalize (< 0: the host build)"""
        K = np.ascontiguousarray(calib6, np.float64).reshape(6)
        self._ck(self.lib.dynoba_builder_set_static_stereo(self.h, _dp(K), float(sigma_px), int(device)))
        self.calib = K.copy()

    def add_static_stereo(self, frame, tracklet, stereo):
        """stereo measurements [n, 3] = (uL, uR, v) of the static tracklets seen at `frame` (uR NaN: no right key-point)"""
        t = np.ascontiguousarray(tracklet, np.int64); z = np.ascontiguousarray(stereo, np.float64).reshape(-1, 3)
        self._ck(self.lib.dynoba_builder_add_static_stereo(self.h, int(frame), t.size, t.ctypes.data_as(c_i64p), _dp(z)))

    def static_stereo_stats(self):
        """dict(added, failed {status: attempts}, never_added) of the stereo landmarks (dynoba_builder_static_stereo_stats)"""
        added = C.c_int64(); never = C.c_int64(); failed = (C.c_int64*4)()
        self._ck(self.lib.dynoba_builder_static_stereo_stats(self.h, C.byref(added), failed, C.byref(never)))
        return dict(added=added.value, failed=list(failed), never_added=never.value)

    def problem(self) -> Problem:
        """the emitted SoA problem as a Problem container"""
        L = self.lib
        npose = C.c_int64(); npt = C.c_int64(); naux = C.c_int64(); nb = C.c_int32()
        self._ck(L.dynoba_builder_counts(self.h, C.byref(npose), C.byref(npt), C.byref(naux), C.byref(nb)))
        pose = np.zeros((npose.value, 12)); point = np.zeros((npt.value, 3)); aux = np.zeros((naux.value, 12))
        order = np.zeros(npose.value, np.int32); pk = np.zeros(npose.value, np.uint64); qk = np.zeros(npt.value, np.uint64)
        self._ck(L.dynoba_builder_get_variables(self.h, _dp(pose), _dp(point), _dp(aux), order.ctypes.data_as(c_ip), pk.ctypes.data_as(c_u64p), qk.ctypes.data_as(c_u64p)))
        blocks = []
        for bi in range(nb.value):
            ty = C.c_int32(); n = C.c_int64(); sd = C.c_int32(); sc = C.c_int64(); k = C.c_double(); ha = C.c_int32()
            self._ck(L.dynoba_builder_block_info(self.h, bi, C.byref(ty), C.byref(n), C.byref(sd), C.byref(sc), C.byref(k), C.byref(ha)))
            idx = np.zeros((n.value, ARITY[ty.value]), np.int32); meas = np.zeros((n.value, max(MEAS_DIM[ty.value], 1)))
            sig = np.zeros(sd.value) if sc.value == 1 else np.zeros((sc.value, sd.value))
            auxi = np.zeros(n.value, np.int32)
            self._ck(L.dynoba_builder_get_block(self.h, bi, idx.ctypes.data_as(c_ip), _dp(meas) if MEAS_DIM[ty.value] else C.cast(None, c_dp), _dp(sig),
                                                auxi.ctypes.data_as(c_ip) if ha.value else C.cast(None, c_ip)))
            blocks.append(FactorBlock(ty.value, idx, meas if MEAS_DIM[ty.value] else None, sig, k.value, auxi if ha.value else None))
        nv = C.c_int64(); nb6 = C.c_int64()
        self._ck(L.dynoba_builder_nav_counts(self.h, C.byref(nv), C.byref(nb6)))
        vel = np.zeros((nv.value, 3)); bias = np.zeros((nb6.value, 6))
        vo = np.zeros(nv.value, np.int32); bo = np.zeros(nb6.value, np.int32)
        self.nav_keys = (np.zeros(nv.value, np.uint64), np.zeros(nb6.value, np.uint64))
        self._ck(L.dynoba_builder_get_nav_variables(self.h, _dp(vel), _dp(bias), vo.ctypes.data_as(c_ip), bo.ctypes.data_as(c_ip),
                                                    self.nav_keys[0].ctypes.data_as(c_u64p), self.nav_keys[1].ctypes.data_as(c_u64p)))
        nav = dict(vel=vel, bias=bias, vel_order=vo, bias_order=bo) if nv.value else {}
        extra = dict(calib=self.calib) if self.calib is not None else {}
        return Problem(pose, point, aux_pose=aux, blocks=blocks, pose_order=order, pose_keys=pk, point_keys=qk, **nav, **extra)

    def emit(self, solver):
        """hand the arrays to a dynosam_b200.binding.Solver handle (no Problem container in between)"""
        self._ck(self.lib.dynoba_builder_emit(self.h, solver.h))
