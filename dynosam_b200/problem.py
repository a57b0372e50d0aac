"""Flat (SoA-friendly) description of a DynOSAM batch problem.

This is the host-side container the C-ABI ingests (include/dynoba.h): variables as dense
arrays, factors as homogeneous blocks.  It plays the role of the reference's
``gtsam::NonlinearFactorGraph`` + ``gtsam::Values`` pair handed to
``LevenbergMarquardtOptimizer`` in ``RegularBackendModule::updateBatch``
(dynosam/src/backend/RegularBackendModule.cc:405-428).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

# factor type ids == include/dynoba.h enum dynoba_factor_type
PRIOR6, BETWEEN6, POSE2POINT3, STEREO3, TERNARY3, HYBRID3, HYBRID_STEREO3, MOTIONPOSE3, \
    SMOOTH_HYBRID6, SMOOTH_POSE6, FLOWPROJ2, PRIOR_VEL3, PRIOR_BIAS6, COMBINED_IMU15, LINEAR_PP3, LINEAR_PPP3 = range(16)
TYPE_NAMES = ["PRIOR6", "BETWEEN6", "POSE2POINT3", "STEREO3", "TERNARY3", "HYBRID3", "HYBRID_STEREO3",
              "MOTIONPOSE3", "SMOOTH_HYBRID6", "SMOOTH_POSE6", "FLOWPROJ2", "PRIOR_VEL3", "PRIOR_BIAS6", "COMBINED_IMU15",
              "LINEAR_PP3", "LINEAR_PPP3"]
ARITY = [1, 2, 2, 2, 3, 3, 3, 4, 3, 3, 2, 1, 1, 6, 2, 3]
DIM = [6, 6, 3, 3, 3, 3, 3, 3, 6, 6, 2, 3, 6, 15, 3, 3]
# LINEAR_PP3 / LINEAR_PPP3 (linearised landmark factors, no noise model: sigma 1): A [3, jcols] row-major | b [3] |
# linearisation point of each pose slot [12] | of the point [3]
MEAS_DIM = [12, 12, 3, 3, 0, 3, 3, 0, 0, 0, 15, 3, 6, 70, 45, 75]
# variable class per key slot: 0 pose(6), 1 point(3), 2 flow(2), 3 velocity(3), 4 IMU bias(6)
SLOT_CLASS = [
    [0], [0, 0], [0, 1], [0, 1], [1, 1, 0], [0, 0, 1], [0, 0, 1], [1, 1, 0, 0], [0, 0, 0], [0, 0, 0], [2, 0],
    [3], [4], [0, 3, 0, 3, 4, 4], [0, 1], [0, 0, 1],
]
CLASS_DIM = [6, 3, 2, 3, 6]
JCOLS = [sum(CLASS_DIM[c] for c in s) for s in SLOT_CLASS]
NEEDS_AUX = [False, False, False, False, False, True, True, False, True, False, False, False, False, False, False, False]
IMU_SQRT_INFO_DIM = 225   # COMBINED_IMU15's sigma: the 15x15 square-root information R, row-major
LINEAR_TYPES = (LINEAR_PP3, LINEAR_PPP3)


def linear_block(type_, idx, A, b, lin_pose, lin_point) -> "FactorBlock":
    """A LINEAR_PP3 / LINEAR_PPP3 block: idx [n, arity], A [n, 3, jcols], b [n, 3], lin_pose [n, npose, 12] (or
    [n, 12] for one pose slot), lin_point [n, 3].  error = 1/2 |A d - b|^2, d = localCoordinates(lin, x)."""
    n, npose = np.asarray(idx).reshape(-1, ARITY[type_]).shape[0], ARITY[type_] - 1
    meas = np.concatenate([np.asarray(A, np.float64).reshape(n, 3*JCOLS[type_]), np.asarray(b, np.float64).reshape(n, 3),
                           np.asarray(lin_pose, np.float64).reshape(n, 12*npose), np.asarray(lin_point, np.float64).reshape(n, 3)], 1)
    return FactorBlock(type_, idx, meas, np.ones(1))


@dataclass
class FactorBlock:
    type: int
    idx: np.ndarray            # int32 [n, arity]
    meas: Optional[np.ndarray]  # float64 [n, meas_dim] or None
    sigma: np.ndarray          # float64 [sigma_dim] (broadcast) or [n, sigma_dim]
    robust_k: float = 0.0      # <= 0: Gaussian; > 0: Huber k
    aux_idx: Optional[np.ndarray] = None  # int32 [n]

    def __post_init__(self):
        self.idx = np.ascontiguousarray(self.idx, dtype=np.int32).reshape(-1, ARITY[self.type])
        n = self.idx.shape[0]
        if MEAS_DIM[self.type]:
            self.meas = np.ascontiguousarray(self.meas, dtype=np.float64).reshape(n, MEAS_DIM[self.type])
        else:
            self.meas = None
        self.sigma = np.ascontiguousarray(self.sigma, dtype=np.float64)
        if self.sigma.ndim == 0:
            self.sigma = self.sigma.reshape(1)
        if self.aux_idx is not None:
            self.aux_idx = np.ascontiguousarray(self.aux_idx, dtype=np.int32).reshape(n)
        if NEEDS_AUX[self.type] and self.aux_idx is None:
            raise ValueError(f"{TYPE_NAMES[self.type]} needs aux_idx")

    @property
    def n(self) -> int:
        return self.idx.shape[0]

    @property
    def sigma_bcast(self) -> bool:
        return self.sigma.ndim == 1

    @property
    def sigma_dim(self) -> int:
        return self.sigma.shape[-1]


@dataclass
class Problem:
    pose: np.ndarray                      # [n_pose, 12]  R row-major | t
    point: np.ndarray                     # [n_point, 3]
    flow: np.ndarray = field(default_factory=lambda: np.zeros((0, 2)))
    aux_pose: np.ndarray = field(default_factory=lambda: np.zeros((0, 12)))
    calib: np.ndarray = field(default_factory=lambda: np.array([721.5377, 721.5377, 0.0, 609.5593, 172.854, 0.5372]))
    blocks: List[FactorBlock] = field(default_factory=list)
    pose_order: Optional[np.ndarray] = None   # int32 [n_pose] ordering hint (frame id)
    pose_keys: Optional[np.ndarray] = None    # uint64 gtsam keys, opaque round-trip
    point_keys: Optional[np.ndarray] = None
    meta: dict = field(default_factory=dict)
    # gtsam::LinearContainerFactor(HessianFactor) priors over pose-like variables (sliding-window marginals): dicts with
    # idx int32[n], lin [n,12], G [6n,6n], g [6n], f over poses; with a "kind" array (POSE6 / VEL3 / BIAS6 per slot) over
    # any pose-like variables, lin packed 12 / 3 / 6 per slot and G, g in the slots' tangent layout (6 / 3 / 6)
    linear_priors: list = field(default_factory=list)
    # navigation variables of visual-inertial graphs: nav-frame velocities [n_vel, 3], IMU biases [n_bias, 6] (acc | gyro),
    # and their ordering hints (frame id), as pose_order is for the poses
    vel: np.ndarray = field(default_factory=lambda: np.zeros((0, 3)))
    bias: np.ndarray = field(default_factory=lambda: np.zeros((0, 6)))
    vel_order: Optional[np.ndarray] = None
    bias_order: Optional[np.ndarray] = None

    def __post_init__(self):
        self.pose = np.ascontiguousarray(self.pose, dtype=np.float64).reshape(-1, 12)
        self.point = np.ascontiguousarray(self.point, dtype=np.float64).reshape(-1, 3)
        self.flow = np.ascontiguousarray(self.flow, dtype=np.float64).reshape(-1, 2)
        self.aux_pose = np.ascontiguousarray(self.aux_pose, dtype=np.float64).reshape(-1, 12)
        self.calib = np.ascontiguousarray(self.calib, dtype=np.float64).reshape(6)
        if self.pose_order is not None:
            self.pose_order = np.ascontiguousarray(self.pose_order, dtype=np.int32)
        self.vel = np.ascontiguousarray(self.vel, dtype=np.float64).reshape(-1, 3)
        self.bias = np.ascontiguousarray(self.bias, dtype=np.float64).reshape(-1, 6)
        for k in ("vel_order", "bias_order"):
            if getattr(self, k) is not None:
                setattr(self, k, np.ascontiguousarray(getattr(self, k), dtype=np.int32))

    @property
    def n_pose(self): return self.pose.shape[0]
    @property
    def n_point(self): return self.point.shape[0]
    @property
    def n_flow(self): return self.flow.shape[0]
    @property
    def n_vel(self): return self.vel.shape[0]
    @property
    def n_bias(self): return self.bias.shape[0]
    @property
    def n_factors(self): return sum(b.n for b in self.blocks)

    def copy(self) -> "Problem":
        return Problem(self.pose.copy(), self.point.copy(), self.flow.copy(), self.aux_pose, self.calib, self.blocks,
                       self.pose_order, self.pose_keys, self.point_keys, dict(self.meta), vel=self.vel.copy(),
                       bias=self.bias.copy(), vel_order=self.vel_order, bias_order=self.bias_order,
                       linear_priors=list(self.linear_priors))

    def jacobian_bytes(self) -> int:
        """Algorithmic bytes of one materialising linearize() (SURVEY.md 8d): every factor record read once,
        every touched variable read once, every whitened Jacobian/rhs element written once."""
        total = 0
        for b in self.blocks:
            rd = 4*ARITY[b.type] + 8*MEAS_DIM[b.type] + 8*b.sigma_dim + (4 if b.aux_idx is not None else 0)
            wr = 8*(DIM[b.type]*JCOLS[b.type] + DIM[b.type])
            total += b.n*(rd + wr)
        total += 96*(self.n_pose + self.aux_pose.shape[0]) + 24*self.n_point + 16*self.n_flow + 24*self.n_vel + 48*self.n_bias
        return total


# ---- gtsam key encoding (dynosam_opt/include/dynosam_opt/Symbols.hpp:14-20,126-152; src/Symbols.cc:160-175)
def symbol_key(c: str, j) -> np.ndarray:
    return (np.uint64(ord(c)) << np.uint64(56)) | np.asarray(j, dtype=np.uint64)


def labeled_symbol_key(c: str, label, j) -> np.ndarray:
    return (np.uint64(ord(c)) << np.uint64(56)) | (np.asarray(label, dtype=np.uint64) << np.uint64(48)) | np.asarray(j, dtype=np.uint64)


def cantor_pair(k1, k2) -> np.ndarray:
    k1 = np.asarray(k1, dtype=np.uint64); k2 = np.asarray(k2, dtype=np.uint64)
    return ((k1 + k2)*(k1 + k2 + np.uint64(1)))//np.uint64(2) + k2


def cantor_depair(z):
    z = np.asarray(z, dtype=np.uint64)
    w = np.floor((np.sqrt(z.astype(np.float64)*8 + 1) - 1)/2).astype(np.uint64)
    t = (w*(w + np.uint64(1)))//np.uint64(2)
    k2 = z - t
    return w - k2, k2


def camera_pose_key(frame): return symbol_key('X', frame)
def velocity_key(frame): return symbol_key('V', frame)
def imu_bias_key(frame): return symbol_key('b', frame)
def static_landmark_key(tracklet): return symbol_key('l', tracklet)
def dynamic_landmark_key(frame, tracklet): return symbol_key('m', cantor_pair(tracklet, frame))
def object_motion_key(obj, frame): return labeled_symbol_key('H', np.asarray(obj, dtype=np.uint64) + np.uint64(ord('0')), frame)
def object_pose_key(obj, frame): return labeled_symbol_key('L', np.asarray(obj, dtype=np.uint64) + np.uint64(ord('0')), frame)
