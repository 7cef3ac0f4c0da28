"""Data association's triangulation on the device.

Drop-in for gtsfm/data_association/data_assoc.py (`DataAssociation`): the same dataclass fields plus `seed`, `device` and
`ctx`.  With GTSfM installed the class subclasses the reference's DataAssociation and overrides `run_triangulation` only,
so `run_triangulation_and_evaluate`, `assemble_gtsfm_data_from_tracks` (largest connected component, metrics, GtsfmData)
and `create_computation_graph` stay the reference's own.  Every track's RANSAC over measurement pairs, its n-view
triangulation and exit code come from one fp64 call into libgtsfm_b200.so (`b2_triangulate_tracks_host`,
csrc/data_assoc.cu).

The device takes NO_RANSAC and RANSAC_SAMPLE_UNIFORM with Cal3Bundler cameras without distortion.  For other inputs
(distorted or other calibrations, the BIASED_BASELINE / TOPK_BASELINES modes) the reference's own `run_triangulation`
runs, logged once; without GTSfM they raise ValueError.  Tracks with more measurement pairs than hypotheses draw their
pairs from a permutation keyed by `seed` and the track's position, not from np.random (csrc/data_assoc_math.cuh).
"""
from __future__ import annotations

import logging
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from .gtsfm_api import (HAVE_GTSFM_DATA_ASSOCIATION, DataAssociation, SfmTrack, TriangulationExitCode, TriangulationOptions,
                        TriangulationSamplingMode)
from .two_view import gt_camera

logger = logging.getLogger(__name__)
_logged_fallback = False

_MODES = {TriangulationSamplingMode.NO_RANSAC.value: _lib.TRI_NO_RANSAC,
          TriangulationSamplingMode.RANSAC_SAMPLE_UNIFORM.value: _lib.TRI_SAMPLE_UNIFORM}
_EXIT = {c.value: c for c in TriangulationExitCode}


def device_camera(cam) -> Optional[tuple]:
    """(R_wTi, t_wTi, f, u0, v0) of a camera the device takes, or None: a gtsam PinholeCameraCal3Bundler with k1 = k2 = 0,
    or such a tuple already."""
    if hasattr(cam, "calibration"):
        cal = cam.calibration()
        if type(cal).__name__ != "Cal3Bundler" or cal.k1() != 0.0 or cal.k2() != 0.0:
            return None
    return gt_camera(cam)


def pack_tracks(tracks_2d: Sequence) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """SfmTrack2d list -> (track_off (T+1,) int64, meas_cam (M,) int64 image indices, meas_uv (M, 2) float64)."""
    lens = np.fromiter((len(t.measurements) for t in tracks_2d), np.int64, count=len(tracks_2d))
    off = np.zeros(len(tracks_2d) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    meas = [m for t in tracks_2d for m in t.measurements]
    cam = np.fromiter((int(m[0]) for m in meas), np.int64, count=len(meas))
    uv = np.array([np.asarray(m[1], np.float64).reshape(2) for m in meas], np.float64).reshape(-1, 2)
    return off, cam, uv


@dataclass(frozen=True)
class B200DataAssociation(DataAssociation):
    """`seed` keys the pair permutation of tracks with more measurement pairs than hypotheses.  `ctx`: a library context,
    or a DeviceFrontEnd whose context to share; by default one is created on `device` at the first call."""

    seed: int = 0
    device: int = 0
    ctx: Any = field(default=None, compare=False, repr=False)

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
        object.__setattr__(self, "ctx", ctx)
        return ctx

    def _mode(self) -> Optional[int]:
        return _MODES.get(getattr(self.triangulation_options.mode, "value", self.triangulation_options.mode))

    def device_params(self) -> "_lib.TriangulationParams":
        """The call's b2_triangulation_params; ValueError for a mode the device does not take."""
        mode = self._mode()
        if mode is None:
            raise ValueError(f"triangulation mode {self.triangulation_options.mode!r} is not served on the device; "
                             f"expected one of {sorted(_MODES)}")
        o = self.triangulation_options
        hyps = min(int(o.num_ransac_hypotheses()), 2 ** 31 - 1) if mode == _lib.TRI_SAMPLE_UNIFORM else 1
        if np.isnan(o.min_triangulation_angle):
            raise ValueError("min_triangulation_angle is NaN")
        return _lib.TriangulationParams(mode, hyps, float(o.reproj_error_threshold), float(o.min_triangulation_angle),
                                        int(self.seed) & (2 ** 64 - 1))

    def triangulate_arrays(self, track_off, meas_cam, meas_uv, cams, cam_valid):
        """The device call on arrays.  track_off (T+1,), meas_cam (M,) image indices < len(cams), meas_uv (M, 2), cams
        (num_images, 15) = R_wTi (row-major), t_wTi, f, u0, v0, cam_valid (num_images,).  -> exit_code (T,) int8,
        point (T, 3) (NaN unless triangulated), avg_error (T,) (NaN for None), inlier (M,) bool."""
        off = np.ascontiguousarray(track_off, np.int64).reshape(-1)
        cam = np.ascontiguousarray(meas_cam, np.int32).reshape(-1)
        uv = np.ascontiguousarray(meas_uv, np.float64).reshape(-1, 2)
        cams = np.ascontiguousarray(cams, np.float64).reshape(-1, 15)
        valid = np.ascontiguousarray(cam_valid, np.uint8).reshape(-1)
        T = len(off) - 1
        if T < 0 or len(cam) != off[-1] or len(uv) != len(cam) or len(valid) != len(cams):
            raise ValueError("track_off, meas_cam, meas_uv, cams and cam_valid do not agree in size")
        ex, pt, avg, inl = np.zeros(T, np.int8), np.empty((T, 3)), np.empty(T), np.zeros(len(cam), np.uint8)
        if T == 0:
            return ex, pt, avg, inl.astype(bool)
        prm = self.device_params()
        ctx = self._context()
        rc = ctx.lib.b2_triangulate_tracks_host(ctx.handle, _lib.ptr(off), T, _lib.ptr(cam), _lib.ptr(uv), _lib.ptr(cams), _lib.ptr(valid),
                                                len(cams), _lib.C.byref(prm), _lib.ptr(ex), _lib.ptr(pt), _lib.ptr(avg), _lib.ptr(inl), None)
        ctx.check(rc, "triangulate_tracks")
        return ex, pt, avg, inl.astype(bool)

    def camera_arrays(self, cameras: Dict[int, Any], num_images: int) -> Optional[Tuple[np.ndarray, np.ndarray]]:
        """{image: camera} -> (cams (num_images, 15), cam_valid), or None when a camera is not one the device takes."""
        cams, valid = np.zeros((num_images, 15)), np.zeros(num_images, np.uint8)
        for i, c in cameras.items():
            if c is None:
                continue
            d = device_camera(c)
            if d is None:
                return None
            R, t, f, u0, v0 = d
            cams[i, :9], cams[i, 9:12], cams[i, 12:] = R.ravel(), t, (f, u0, v0)
            valid[i] = 1
        return cams, valid

    def run_triangulation(self, cameras: Dict[int, Any], tracks_2d: List) -> Tuple[List[Optional[Any]], List[Optional[float]], List]:
        """The reference's three lists: SfmTrack (the inlier measurements in track order) or None, the average
        reprojection error or None, and the TriangulationExitCode of every track, in input order."""
        if len(cameras) == 0 or len(tracks_2d) == 0:
            logger.warning("No cameras or no tracks found, skipping triangulation.")
            return [], [], []
        off, img, uv = pack_tracks(tracks_2d)
        num_images = int(max(max(cameras), img.max(initial=-1))) + 1
        if min(cameras) < 0 or img.min(initial=0) < 0:
            raise ValueError("image indices must be >= 0")
        arr = self.camera_arrays(cameras, num_images) if self._mode() is not None else None
        if arr is None:
            if not HAVE_GTSFM_DATA_ASSOCIATION:
                raise ValueError("the device takes NO_RANSAC / RANSAC_SAMPLE_UNIFORM with undistorted Cal3Bundler cameras only, "
                                 "and GTSfM is not installed to run the reference for the rest")
            global _logged_fallback
            if not _logged_fallback:
                logger.info("B200DataAssociation: mode or calibration not served on the device; running the reference's triangulation")
                _logged_fallback = True
            return super().run_triangulation(cameras, tracks_2d)
        ex, pt, avg, inl = self.triangulate_arrays(off, img, uv, *arr)
        return unpack(tracks_2d, off, ex, pt, avg, inl)


def unpack(tracks_2d, off, ex, pt, avg, inl):
    """Device arrays -> the reference's (sfm_tracks, avg_track_reproj_errors, triangulation_exit_codes)."""
    tracks, errs, codes = [], [], []
    for t, tr in enumerate(tracks_2d):
        code = _EXIT[int(ex[t])]
        codes.append(code)
        errs.append(None if np.isnan(avg[t]) else float(avg[t]))
        if code != TriangulationExitCode.SUCCESS:
            tracks.append(None)
            continue
        s = SfmTrack(pt[t])
        for k in np.flatnonzero(inl[off[t]:off[t + 1]]):
            i, uv = tr.measurements[k]
            s.addMeasurement(i, uv)
        tracks.append(s)
    return tracks, errs, codes
