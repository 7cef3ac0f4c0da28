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
