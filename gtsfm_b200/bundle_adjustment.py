"""Global bundle adjustment on the device.

Drop-in for gtsfm/bundle/bundle_adjustment.py (`BundleAdjustmentOptimizer`): the same constructor plus `device` and `ctx`.
With GTSfM installed the class subclasses the reference's optimizer and overrides `run_ba_stage_with_filtering` only, so
`run_ba`'s stage loop, `evaluate`, the Sim(3) alignment and the metrics stay the reference's own.  The optimisation itself
(gtsam's Levenberg-Marquardt over every camera pose, calibration and point) is one fp64 call into libgtsfm_b200.so
(`b2_bundle_adjust_host`, csrc/global_ba.cu); the result is written into a gtsam.Values and goes through the reference's
own GtsfmData.from_values and filter_landmarks.

The device serves the configs' graph: Cal3Bundler cameras with their own calibrations (shared_calib False), HUBER or
NONE, the Karcher gauge or the first-pose prior, calibration priors.  Other inputs (GNC or GMC, shared_calib,
relative_pose_priors, use_pose_prior, use_first_point_prior, use_calibration_prior False, other calibrations,
allow_indeterminate_linear_system False with two cameras, a problem over the "ba_workspace_mb" budget) run the reference's
own method, logged once; without GTSfM they raise ValueError.
"""
from __future__ import annotations

import logging
from typing import Any, Optional

import numpy as np

from . import _lib
from .gtsfm_api import HAVE_GTSFM_BA, BundleAdjustmentOptimizer, RobustBAMode

logger = logging.getLogger(__name__)
_logged_fallback = False
DEFAULT_WORKSPACE_MB = 4096  # b2_context's "ba_workspace_mb" default
GTSAM_MAX_ITERS = 100        # gtsam.LevenbergMarquardtParams().maxIterations


class B200BundleAdjustmentOptimizer(BundleAdjustmentOptimizer):
    """`ctx`: a library context, or a DeviceFrontEnd whose context to share; by default one is created on `device` at the
    first call."""

    def __init__(self, *args, device: int = 0, ctx: Any = None, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.device = device
        self.ctx = ctx

    def __getstate__(self):  # device state is created lazily on the worker, like the other plugins
        d = dict(self.__dict__)
        d["ctx"] = None
        return d

    def __setstate__(self, d):
        self.__dict__.update(d)

    def _context(self) -> _lib.Context:
        ctx = getattr(self.ctx, "ctx", self.ctx)
        if ctx is None:
            ctx = _lib.Context(self.device)
        self.ctx = ctx
        return ctx

    def _mode(self):
        m = self._robust_ba_mode
        return RobustBAMode[m] if isinstance(m, str) else m

    def unserved(self, relative_pose_priors=None) -> Optional[str]:
        """Why the settings are not served on the device, or None."""
        if self._use_gnc:
            return "use_gnc"
        if self._mode().value not in ("NONE", "HUBER"):
            return f"robust_ba_mode {self._mode().value}"
        if self._shared_calib:
            return "shared_calib"
        if relative_pose_priors:
            return "relative_pose_priors"
        if self._use_karcher_mean_factor and self._use_pose_prior:
            return "use_pose_prior"
        if self._use_first_point_prior:
            return "use_first_point_prior"
        if not self._use_calibration_prior:
            return "use_calibration_prior False"
        return None

    def device_params(self) -> _lib.BaParams:
        """The call's b2_ba_params; ValueError for settings the device does not serve."""
        why = self.unserved()
        if why is not None:
            raise ValueError(f"{why} is not served on the device")
        p = _lib.BaParams()
        p.noise_sigma = float(self._measurement_noise_sigma)
        p.huber_k = float(self._robust_noise_basin) if self._mode().value == "HUBER" else 0.0
        p.gauge = _lib.BA_KARCHER if self._use_karcher_mean_factor else _lib.BA_FIRST_POSE_PRIOR
        p.max_iters = int(self._max_iterations) if self._max_iterations else GTSAM_MAX_ITERS
        p.karcher_beta = 1000.0  # KarcherMeanFactorPose3(keys, 6, 1000)
        p.pose_prior_sigma = float(self._cam_pose3_prior_noise_sigma)
        p.cal_prior_sigma[:] = (float(self._calibration_prior_focal_sigma), float(self._calibration_prior_dist_sigma),
                                float(self._calibration_prior_dist_sigma))
        return p

    def fits(self, num_cameras: int, track_off) -> bool:
        """Whether the problem's device workspace is within the context's "ba_workspace_mb"."""
        off = np.ascontiguousarray(track_off, np.int64).reshape(-1)
        lib = _lib.load()
        need = lib.b2_bundle_adjust_workspace_bytes(int(num_cameras), len(off) - 1, _lib.ptr(off))
        ctx = getattr(self.ctx, "ctx", self.ctx)
        mb = ctx.options.get("ba_workspace_mb", DEFAULT_WORKSPACE_MB) if ctx is not None else DEFAULT_WORKSPACE_MB
        return 0 < need <= mb << 20

    def adjust_arrays(self, cams, points, track_off, meas_cam, meas_uv, trace: bool = False):
        """The device call on arrays.  cams (C, 17) = R_wTi (row-major), t_wTi, f, k1, k2, u0, v0 of the modelled cameras in
        order; points (N, 3); track_off (N + 1,); meas_cam (M,) indices into cams; meas_uv (M, 2).  -> dict of cams,
        points, reproj_err (M,) (NaN behind the camera), final_error, iterations and, with `trace`, trace and trials."""
        cams = np.ascontiguousarray(cams, np.float64).reshape(-1, 17)
        pts = np.ascontiguousarray(points, np.float64).reshape(-1, 3)
        off = np.ascontiguousarray(track_off, np.int64).reshape(-1)
        cam = np.ascontiguousarray(meas_cam, np.int32).reshape(-1)
        uv = np.ascontiguousarray(meas_uv, np.float64).reshape(-1, 2)
        if len(off) != len(pts) + 1 or off[-1] != len(cam) or len(uv) != len(cam):
            raise ValueError("points, track_off, meas_cam and meas_uv do not agree in size")
        prm = self.device_params()
        ctx = self._context()
        C, N, M = len(cams), len(pts), len(cam)
        cams_out, pts_out, err = np.empty_like(cams), np.empty_like(pts), np.empty(M)
        res = _lib.BaResult()
        tr = np.zeros(prm.max_iters + 2) if trace else None
        cap = 64 * (prm.max_iters + 2) if trace else 0
        trials = np.zeros(cap, np.int32) if trace else None
        rc = ctx.lib.b2_bundle_adjust_host(ctx.handle, C, _lib.ptr(cams), N, _lib.ptr(pts), _lib.ptr(off), _lib.ptr(cam), _lib.ptr(uv),
                                           _lib.C.byref(prm), _lib.ptr(cams_out), _lib.ptr(pts_out), _lib.ptr(err), _lib.C.byref(res),
                                           _lib.ptr(tr), _lib.ptr(trials), cap, None)
        ctx.check(rc, "bundle_adjust")
        out = dict(cams=cams_out, points=pts_out, reproj_err=err, final_error=float(res.final_error), iterations=int(res.iterations))
        if trace:
            out["trace"] = tr[:res.trace_len].copy()
            out["trials"] = trials[:min(res.trials, cap)].copy()
        return out

    def run_ba_stage_with_filtering(self, initial_data, absolute_pose_priors, relative_pose_priors, reproj_error_thresh,
                                    verbose: bool = True):
        """The reference's (optimized_data, filtered_data, valid_mask, final_error) with the optimisation on the device."""
        packed = None
        why = self.unserved(relative_pose_priors)
        if why is None and HAVE_GTSFM_BA:
            if initial_data.number_tracks() == 0 or len(initial_data.get_valid_camera_indices()) == 0:
                return initial_data, initial_data, [False] * initial_data.number_tracks(), 0.0
            if not self._allow_indeterminate_linear_system and self.is_two_view_ba(initial_data):
                why = "allow_indeterminate_linear_system False with two cameras"
            else:
                packed = pack_gtsfm_data(initial_data)
                if packed is None:
                    why = "a calibration other than Cal3Bundler, or a track without a modelled camera"
                elif not self.fits(len(packed[0]), packed[3]):
                    why = "the problem is over the ba_workspace_mb budget"
        if packed is None:
            if not HAVE_GTSFM_BA:
                raise ValueError(f"{why or 'GtsfmData'} needs the reference's BundleAdjustmentOptimizer, and GTSfM is not installed")
            global _logged_fallback
            if not _logged_fallback:
                logger.info("B200BundleAdjustmentOptimizer: %s is not served on the device; running the reference's method", why)
                _logged_fallback = True
            return super().run_ba_stage_with_filtering(initial_data, absolute_pose_priors, relative_pose_priors,
                                                       reproj_error_thresh, verbose)
        model, cams, pts, off, cam, uv = packed
        out = self.adjust_arrays(cams, pts, off, cam, uv)
        optimized_data = unpack_to_gtsfm_data(initial_data, model, out)
        if reproj_error_thresh is not None:
            filtered, valid_mask = optimized_data.filter_landmarks(reproj_error_thresh)
        else:
            filtered, valid_mask = optimized_data, [True] * optimized_data.number_tracks()
        return optimized_data, filtered, valid_mask, out["final_error"]


def pack_gtsfm_data(data):  # pragma: no cover - needs gtsam
    """GtsfmData -> (modelled camera ids, cams (C, 17), points, track_off, meas_cam, meas_uv), the reprojection factors the
    reference builds (measurements in cameras outside the model are not factors), or None when a camera is not a
    Cal3Bundler or a track has no factor."""
    model = sorted(data.get_valid_camera_indices())
    slot = {i: a for a, i in enumerate(model)}
    cams = np.zeros((len(model), 17))
    for a, i in enumerate(model):
        c = data.get_camera(i)
        k = c.calibration()
        if type(k).__name__ != "Cal3Bundler":
            return None
        p = c.pose()
        cams[a, :9], cams[a, 9:12] = p.rotation().matrix().ravel(), p.translation()
        cams[a, 12:] = (k.fx(), k.k1(), k.k2(), k.px(), k.py())
    off, cam, uv, pts = [0], [], [], []
    for j in range(data.number_tracks()):
        t = data.get_track(j)
        for k in range(t.numberMeasurements()):
            i, m = t.measurement(k)
            if i in slot:
                cam.append(slot[i])
                uv.append(np.asarray(m, float).reshape(2))
        if len(cam) == off[-1]:
            return None
        off.append(len(cam))
        pts.append(np.asarray(t.point3(), float).reshape(3))
    return model, cams, np.array(pts), np.array(off, np.int64), np.array(cam, np.int32), np.array(uv, float).reshape(-1, 2)


def unpack_to_gtsfm_data(initial_data, model, out):  # pragma: no cover - needs gtsam
    """The device result as a gtsam.Values through the reference's own GtsfmData.from_values."""
    import gtsam
    from gtsam.symbol_shorthand import K, P, X
    from gtsfm.common.gtsfm_data import GtsfmData

    values = gtsam.Values()
    for a, i in enumerate(model):
        c = out["cams"][a]
        values.insert(X(i), gtsam.Pose3(gtsam.Rot3(c[:9].reshape(3, 3)), c[9:12]))
        values.insert(K(i), gtsam.Cal3Bundler(c[12], c[13], c[14], c[15], c[16]))
    for j, p in enumerate(out["points"]):
        values.insert(P(j), np.asarray(p, float))
    return GtsfmData.from_values(values, initial_data, False)
