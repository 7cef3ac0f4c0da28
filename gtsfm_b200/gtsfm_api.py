"""The reference's plugin API, re-used when GTSfM is importable and mirrored when it is not.

Inside a GTSfM environment the plugins subclass the reference's own abstract bases so they drop into
scene_optimizer.py through a Hydra `_target_` swap (SURVEY.md §8b):

  * gtsfm/frontend/detector_descriptor/detector_descriptor_base.py:19-57   DetectorDescriptorBase
  * gtsfm/frontend/matcher/matcher_base.py:15-67                            MatcherBase
  * gtsfm/frontend/verifier/verifier_base.py:20-90                          VerifierBase
  * gtsfm/common/keypoints.py:15-231  Keypoints ;  gtsfm/common/image.py:19-41  Image

On a box without gtsfm / gtsam / dask (the GPU test boxes) the same names resolve to the minimal mirrors below:
same constructor arguments, attributes, method signatures and failure values, nothing else.
"""
from __future__ import annotations

import abc
import copy
from typing import Optional, Tuple

import numpy as np

try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsfm.common.image import Image
    from gtsfm.common.keypoints import Keypoints
    from gtsfm.frontend.detector_descriptor.detector_descriptor_base import DetectorDescriptorBase
    from gtsfm.frontend.matcher.matcher_base import MatcherBase
    from gtsfm.frontend.verifier.verifier_base import VerifierBase

    try:  # the retriever base drags in gtsfm.evaluation.metrics -> h5py / open3d: optional on its own
        from gtsfm.retriever.retriever_base import RetrieverBase
    except Exception:  # noqa: BLE001
        RetrieverBase = None
    try:
        from gtsfm.frontend.global_descriptor.global_descriptor_base import GlobalDescriptorBase
    except Exception:  # noqa: BLE001
        GlobalDescriptorBase = None
    HAVE_GTSFM = True
except Exception:  # noqa: BLE001 - any import problem (gtsam, dask, hydra ...) means "not a GTSfM environment"
    HAVE_GTSFM = False

    class Keypoints:  # mirrors gtsfm/common/keypoints.py:15-127
        def __init__(self, coordinates: np.ndarray, scales: Optional[np.ndarray] = None, responses: Optional[np.ndarray] = None):
            self.coordinates = coordinates
            self.scales = scales
            self.responses = responses

        def __len__(self) -> int:
            return self.coordinates.shape[0]

        def __eq__(self, other: object) -> bool:
            if not isinstance(other, Keypoints):
                return False

            def same(a, b):
                if a is None and b is None:
                    return True
                return a is not None and b is not None and np.array_equal(a, b)

            return np.array_equal(self.coordinates, other.coordinates) and same(self.scales, other.scales) and same(self.responses, other.responses)

        def __ne__(self, other: object) -> bool:
            return not self == other

        def extract_indices(self, indices: np.ndarray) -> "Keypoints":
            if indices.size == 0:
                return Keypoints(coordinates=np.zeros(shape=(0, 2)))
            return Keypoints(self.coordinates[indices], None if self.scales is None else self.scales[indices],
                             None if self.responses is None else self.responses[indices])

        def get_top_k(self, k: int) -> Tuple["Keypoints", np.ndarray]:
            if k >= len(self):
                return copy.deepcopy(self), np.arange(len(self))
            if self.responses is None:
                sel = np.arange(k, dtype=np.uint32)
            else:
                sel = np.argpartition(-self.responses, k)[:k]
            return self.extract_indices(sel), sel

        def filter_by_mask(self, mask: np.ndarray) -> Tuple["Keypoints", np.ndarray]:
            r = np.round(self.coordinates).astype(int)
            valid = np.flatnonzero(mask[r[:, 1], r[:, 0]] == 1)
            return self.extract_indices(valid), valid

    class Image:  # mirrors gtsfm/common/image.py:19-41 (the fields the hot path touches)
        def __init__(self, value_array: np.ndarray, exif_data=None, file_name: Optional[str] = None, mask: Optional[np.ndarray] = None):
            self.value_array = value_array
            self.exif_data = exif_data
            self.file_name = file_name
            self.mask = mask

        @property
        def height(self) -> int:
            return self.value_array.shape[0]

        @property
        def width(self) -> int:
            return self.value_array.shape[1]

        @property
        def shape(self):
            return self.value_array.shape

    class DetectorDescriptorBase(abc.ABC):
        def __init__(self, max_keypoints: int = 5000):
            self.max_keypoints = max_keypoints

        @abc.abstractmethod
        def detect_and_describe(self, image: Image) -> Tuple[Keypoints, np.ndarray]:
            ...

    class MatcherBase(abc.ABC):
        @abc.abstractmethod
        def match(self, keypoints_i1, keypoints_i2, descriptors_i1, descriptors_i2, im_shape_i1, im_shape_i2) -> np.ndarray:
            ...

    RetrieverBase = None
    GlobalDescriptorBase = None

    NUM_MATCHES_REQ_E_MATRIX = 5
    NUM_MATCHES_REQ_F_MATRIX = 8

    class VerifierBase(abc.ABC):
        def __repr__(self) -> str:
            return f"{type(self).__name__}__use_intrinsics{self._use_intrinsics_in_verification}_{self._estimation_threshold_px}px"

        def __init__(self, use_intrinsics_in_verification: bool, estimation_threshold_px: float) -> None:
            self._use_intrinsics_in_verification = use_intrinsics_in_verification
            self._estimation_threshold_px = estimation_threshold_px
            self._min_matches = NUM_MATCHES_REQ_E_MATRIX if use_intrinsics_in_verification else NUM_MATCHES_REQ_F_MATRIX
            self._failure_result = (None, None, np.array([], dtype=np.uint64), 0.0)

        @abc.abstractmethod
        def verify(self, keypoints_i1, keypoints_i2, match_indices, camera_intrinsics_i1, camera_intrinsics_i2):
            ...


try:  # pragma: no cover
    from gtsam import Cal3Bundler, Rot3, Unit3

    HAVE_GTSAM = True
except Exception:  # noqa: BLE001
    HAVE_GTSAM = False

    class Rot3:  # the subset of gtsam.Rot3 the verifier's callers use
        def __init__(self, R: Optional[np.ndarray] = None):
            self._R = np.eye(3) if R is None else np.asarray(R, np.float64).reshape(3, 3)

        def matrix(self) -> np.ndarray:
            return self._R.copy()

        def inverse(self) -> "Rot3":
            return Rot3(self._R.T)

        def between(self, other: "Rot3") -> "Rot3":
            return Rot3(self._R.T @ other._R)

    class Unit3:
        def __init__(self, v: Optional[np.ndarray] = None):
            v = np.array([1.0, 0, 0]) if v is None else np.asarray(v, np.float64).ravel()
            self._v = v / np.linalg.norm(v)

        def point3(self) -> np.ndarray:
            return self._v.copy()

    class Cal3Bundler:
        def __init__(self, fx: float = 1.0, k1: float = 0.0, k2: float = 0.0, u0: float = 0.0, v0: float = 0.0):
            self._f, self._k1, self._k2, self._u0, self._v0 = float(fx), float(k1), float(k2), float(u0), float(v0)

        def fx(self):
            return self._f

        def k1(self):
            return self._k1

        def k2(self):
            return self._k2

        def px(self):
            return self._u0

        def py(self):
            return self._v0

        def K(self) -> np.ndarray:
            return np.array([[self._f, 0, self._u0], [0, self._f, self._v0], [0, 0, 1.0]])

        def calibrate(self, p: np.ndarray) -> np.ndarray:
            p = np.asarray(p, np.float64).ravel()
            x, y = (p[0] - self._u0) / self._f, (p[1] - self._v0) / self._f
            if self._k1 == 0.0 and self._k2 == 0.0:
                return np.array([x, y])
            xu, yu = x, y
            for _ in range(20):  # fixed-point undistortion
                r2 = xu * xu + yu * yu
                g = 1 + self._k1 * r2 + self._k2 * r2 * r2
                xu, yu = x / g, y / g
            return np.array([xu, yu])


if RetrieverBase is None:

    class RetrieverBase(abc.ABC):  # mirrors gtsfm/retriever/retriever_base.py:17-60
        def set_max_frame_lookahead(self, n) -> None:
            raise AttributeError(f"{type(self).__name__} has no max_frame_lookahead")

        def set_num_matched(self, n) -> None:
            raise AttributeError(f"{type(self).__name__} has no num_matched")

        @abc.abstractmethod
        def get_image_pairs(self, global_descriptors, image_fnames, plots_output_dir=None):
            ...

        def save_diagnostics(self, image_fnames, pairs, plots_output_dir) -> None:
            return None


if GlobalDescriptorBase is None:

    class GlobalDescriptorBase:  # mirrors gtsfm/frontend/global_descriptor/global_descriptor_base.py:14-47
        @abc.abstractmethod
        def describe_batch(self, images):
            ...

        @abc.abstractmethod
        def get_preprocessing_transforms(self):
            ...


try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsfm.common.two_view_estimation_report import TwoViewEstimationReport
except Exception:  # noqa: BLE001
    from dataclasses import dataclass

    @dataclass(frozen=False)
    class TwoViewEstimationReport:  # mirrors gtsfm/common/two_view_estimation_report.py:13-56 (fields and defaults)
        v_corr_idxs: np.ndarray
        num_inliers_est_model: float
        inlier_ratio_est_model: Optional[float] = None
        num_inliers_gt_model: Optional[float] = None
        inlier_ratio_gt_model: Optional[float] = None
        v_corr_idxs_inlier_mask_gt: Optional[np.ndarray] = None
        R_error_deg: Optional[float] = None
        U_error_deg: Optional[float] = None
        i2Ri1: Optional[Rot3] = None
        i2Ui1: Optional[Unit3] = None
        reproj_error_gt_model: Optional[np.ndarray] = None
        inlier_avg_reproj_error_gt_model: Optional[float] = None
        outlier_avg_reproj_error_gt_model: Optional[float] = None


try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsfm.view_graph_estimator.cycle_consistent_rotation_estimator import EdgeErrorAggregationCriterion
    from gtsfm.view_graph_estimator.view_graph_estimator_base import ViewGraphEstimatorBase
except Exception:  # noqa: BLE001
    from enum import Enum

    class EdgeErrorAggregationCriterion(str, Enum):  # mirrors cycle_consistent_rotation_estimator.py:33-48
        MIN_EDGE_ERROR = "MIN_EDGE_ERROR"
        MEDIAN_EDGE_ERROR = "MEDIAN_EDGE_ERROR"

    class ViewGraphEstimatorBase(abc.ABC):  # the part of view_graph_estimator_base.py:38-92 that `run` needs
        @abc.abstractmethod
        def run(self, i2Ri1_dict, i2Ui1_dict, calibrations, corr_idxs_i1i2, keypoints, two_view_reports, output_dir=None):
            ...


try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsam import SfmTrack
    from gtsfm.common.sfm_track import SfmMeasurement, SfmTrack2d
    from gtsfm.data_association.data_assoc import DataAssociation
    from gtsfm.data_association.point3d_initializer import TriangulationExitCode, TriangulationOptions, TriangulationSamplingMode
    HAVE_GTSFM_DATA_ASSOCIATION = True  # the reference's DataAssociation is the base: its run_triangulation is the fallback
except Exception:  # noqa: BLE001
    HAVE_GTSFM_DATA_ASSOCIATION = False
    import sys
    from dataclasses import dataclass
    from enum import Enum
    from typing import List, NamedTuple

    class TriangulationExitCode(Enum):  # mirrors point3d_initializer.py:34-43
        SUCCESS = 0
        CHEIRALITY_FAILURE = 1
        INLIERS_UNDERCONSTRAINED = 2
        POSES_UNDERCONSTRAINED = 3
        EXCEEDS_REPROJ_THRESH = 4
        LOW_TRIANGULATION_ANGLE = 5

    class TriangulationSamplingMode(str, Enum):  # mirrors point3d_initializer.py:46-58
        NO_RANSAC = "NO_RANSAC"
        RANSAC_SAMPLE_UNIFORM = "RANSAC_SAMPLE_UNIFORM"
        RANSAC_SAMPLE_BIASED_BASELINE = "RANSAC_SAMPLE_BIASED_BASELINE"
        RANSAC_TOPK_BASELINES = "RANSAC_TOPK_BASELINES"

    class TriangulationOptions(NamedTuple):  # mirrors point3d_initializer.py:61-112
        mode: TriangulationSamplingMode
        reproj_error_threshold: float = np.inf
        min_triangulation_angle: float = 0.0
        min_inlier_ratio: float = 0.1
        confidence: float = 0.9999
        dyn_num_hypotheses_multiplier: float = 3.0
        min_num_hypotheses: int = 0
        max_num_hypotheses: int = sys.maxsize

        def num_ransac_hypotheses(self) -> int:
            assert self.reproj_error_threshold > 0
            assert 0 < self.min_inlier_ratio < 1
            assert 0 < self.confidence < 1
            assert self.dyn_num_hypotheses_multiplier > 0
            assert 0 <= self.min_num_hypotheses < self.max_num_hypotheses
            dyn = int((np.log(1 - self.confidence) / np.log(1 - self.min_inlier_ratio ** 2)) * self.dyn_num_hypotheses_multiplier)
            return max(min(self.max_num_hypotheses, dyn), self.min_num_hypotheses)

    class SfmMeasurement(NamedTuple):  # mirrors gtsfm/common/sfm_track.py:18-35
        i: int
        uv: np.ndarray

    class SfmTrack2d(NamedTuple):  # mirrors gtsfm/common/sfm_track.py:38-78 (what triangulation reads)
        measurements: List[SfmMeasurement]

        def number_measurements(self) -> int:
            return len(self.measurements)

        def measurement(self, idx: int) -> SfmMeasurement:
            return self.measurements[idx]

    class SfmTrack:  # the part of gtsam.SfmTrack a triangulated track exposes
        def __init__(self, pt):
            self._pt = np.asarray(pt, np.float64).reshape(3)
            self._meas: list = []

        def addMeasurement(self, i, uv) -> None:  # noqa: N802 - gtsam's name
            self._meas.append((int(i), np.asarray(uv, np.float64).reshape(2)))

        def numberMeasurements(self) -> int:  # noqa: N802
            return len(self._meas)

        def measurement(self, k):
            return self._meas[k]

        def point3(self) -> np.ndarray:
            return self._pt

    @dataclass(frozen=True)
    class DataAssociation:  # the fields of data_assoc.py:45-58 and the method a subclass overrides
        min_track_len: int
        triangulation_options: TriangulationOptions
        save_track_patches_viz: Optional[bool] = False

        def run_triangulation(self, cameras, tracks_2d):
            raise NotImplementedError("the reference's run_triangulation needs GTSfM")


try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsfm.averaging.translation.averaging_1dsfm import TranslationAveraging1DSFM
    HAVE_GTSFM_1DSFM = True  # the reference's class is the base: its sampler and run_translation_averaging are used
except Exception:  # noqa: BLE001
    HAVE_GTSFM_1DSFM = False
    from enum import Enum

    class TranslationAveraging1DSFM:  # mirrors averaging_1dsfm.py:79-155 (constructor, sampler; no averaging)
        class ProjectionSamplingMethod(str, Enum):
            SAMPLE_INPUT_MEASUREMENTS = "SAMPLE_INPUT_MEASUREMENTS"
            SAMPLE_WITH_INPUT_DENSITY = "SAMPLE_WITH_INPUT_DENSITY"
            SAMPLE_WITH_UNIFORM_DENSITY = "SAMPLE_WITH_UNIFORM_DENSITY"

        def __init__(self, robust_measurement_noise: bool = True, use_tracks_for_averaging: bool = True,
                     reject_outliers: bool = True, projection_sampling_method=ProjectionSamplingMethod.SAMPLE_WITH_UNIFORM_DENSITY,
                     max_delayed_calls: int = 16, use_all_tracks_for_averaging: bool = False,
                     use_relative_camera_poses: bool = True) -> None:
            self._robust_measurement_noise = robust_measurement_noise
            self._max_1dsfm_projection_directions = 2000
            self._outlier_weight_threshold = 0.125
            self._reject_outliers = reject_outliers
            self._projection_sampling_method = projection_sampling_method
            self._use_tracks_for_averaging = use_tracks_for_averaging
            self._max_delayed_calls = max_delayed_calls
            self._use_relative_camera_poses = use_relative_camera_poses
            self._use_all_tracks_for_averaging = use_all_tracks_for_averaging
            np.random.seed(0)

        def __sample_projection_directions(self, w_i2Ui1_list):
            """The reference's sampler on NumPy's global RNG, as (K, 3) rows normalised as gtsam's Unit3 (Eigen) does."""
            method = self.ProjectionSamplingMethod(self._projection_sampling_method)
            num = self._max_1dsfm_projection_directions
            if method == self.ProjectionSamplingMethod.SAMPLE_INPUT_MEASUREMENTS:
                n = len(w_i2Ui1_list)
                return [w_i2Ui1_list[i] for i in np.random.choice(n, min(n, num), replace=False)]
            if method == self.ProjectionSamplingMethod.SAMPLE_WITH_UNIFORM_DENSITY:
                v = np.random.normal(size=(num, 3))
                return v / np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])[:, None]
            raise ValueError("SAMPLE_WITH_INPUT_DENSITY samples a scipy KDE through GTSfM, which is not installed")

        def run_translation_averaging(self, *args, **kwargs):
            raise NotImplementedError("run_translation_averaging (track selection, TranslationRecovery) needs GTSfM")


try:  # pragma: no cover - exercised only inside a full GTSfM environment
    from gtsfm.bundle.bundle_adjustment import BundleAdjustmentOptimizer, RobustBAMode
    HAVE_GTSFM_BA = True  # the reference's class is the base: its stage loop, evaluate and fallback are used
except Exception:  # noqa: BLE001
    HAVE_GTSFM_BA = False
    from enum import Enum

    class RobustBAMode(Enum):  # mirrors bundle_adjustment.py:44-51
        NONE = "NONE"
        HUBER = "HUBER"
        GMC = "GMC"
        TLS = "TLS"

    class BundleAdjustmentOptimizer:  # mirrors bundle_adjustment.py:64-143 (the constructor's fields; no graph, no metrics)
        def __init__(self, reproj_error_thresholds=(None,), robust_ba_mode=RobustBAMode.NONE, shared_calib: bool = False,
                     max_iterations: Optional[int] = None, cam_pose3_prior_noise_sigma: float = 0.1,
                     calibration_prior_focal_sigma: float = 20.0, calibration_prior_dist_sigma: float = 0.1,
                     measurement_noise_sigma: float = 2.0, allow_indeterminate_linear_system: bool = True,
                     print_summary: bool = False, ordering_type: str = "METIS", save_iteration_visualization: bool = False,
                     robust_noise_basin: float = 1.345, use_karcher_mean_factor: bool = True, use_pose_prior: bool = False,
                     use_calibration_prior: bool = True, use_first_point_prior: bool = False, use_gnc: bool = False,
                     gnc_loss=RobustBAMode.GMC, factor_weight_outlier_threshold: float = 0.0, min_track_length: int = 2) -> None:
            self._reproj_error_thresholds = reproj_error_thresholds
            self._robust_ba_mode = RobustBAMode[robust_ba_mode] if isinstance(robust_ba_mode, str) else robust_ba_mode
            self._shared_calib = shared_calib
            self._max_iterations = max_iterations
            self._cam_pose3_prior_noise_sigma = cam_pose3_prior_noise_sigma
            self._use_calibration_prior = use_calibration_prior
            self._calibration_prior_focal_sigma = calibration_prior_focal_sigma
            self._calibration_prior_dist_sigma = calibration_prior_dist_sigma
            self._measurement_noise_sigma = measurement_noise_sigma
            self._allow_indeterminate_linear_system = allow_indeterminate_linear_system
            self._ordering_type = ordering_type
            self._print_summary = print_summary
            self._save_iteration_visualization = save_iteration_visualization
            self._robust_noise_basin = robust_noise_basin
            self._use_karcher_mean_factor = use_karcher_mean_factor
            self._use_pose_prior = use_pose_prior
            self._use_first_point_prior = use_first_point_prior
            self._use_gnc = use_gnc
            self._gnc_loss = RobustBAMode[gnc_loss] if isinstance(gnc_loss, str) else gnc_loss
            self._factor_weight_outlier_threshold = factor_weight_outlier_threshold
            self._min_track_length = min_track_length

        def run_ba_stage_with_filtering(self, *args, **kwargs):
            raise NotImplementedError("the reference's run_ba_stage_with_filtering needs GTSfM")
