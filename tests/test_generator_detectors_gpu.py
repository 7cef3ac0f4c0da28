"""GPU: B200CorrespondenceGenerator with the SIFT, ORB and D2-Net detectors and the two-way matcher, and with SuperPoint and
SuperGlue, returns what the per-image and per-pair plugins return for the same images: the keypoints and descriptors of
`detect_and_describe` (as sets: the device top-k keeps its own order), the match rows of `match` on the generator's own
features in the plugin's dtype, and the two-view results of B200Ransac.verify_many.  The job mixes two image shapes, a masked
image and a flat image (no SIFT or ORB keypoints: its pairs give the reference's empty matches and the verifier's failure)."""
import numpy as np
import pytest
import torch

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator
from gtsfm_b200.detector_descriptor import (B200D2NetDetectorDescriptor, B200ORBDetectorDescriptor, B200SIFTDetectorDescriptor,
                                            B200SuperPointDetectorDescriptor)
from gtsfm_b200.gtsfm_api import Cal3Bundler, Image, Keypoints
from gtsfm_b200.matcher import B200SuperGlueMatcher, B200TwoWayMatcher
from gtsfm_b200.verifier import B200Ransac

pytestmark = pytest.mark.gpu

K = 1500
RATIO = 0.8
PAIRS = [(0, 1), (1, 2), (0, 2), (2, 3), (3, 4), (4, 5), (0, 5)]  # (2, 3) spans the two shapes; image 5 is flat


def _job(golden_dir):
    lund = np.load(golden_dir / "lund_door_images.npz")
    a = [np.ascontiguousarray(lund[f"gray_{i}"][250:810, 20:740]) for i in (1, 2, 3)]  # 560 x 720
    b = [np.ascontiguousarray(lund[f"gray_{i}"][300:780, 60:700]) for i in (4, 5)]  # 480 x 640
    mask = np.zeros(a[2].shape, np.uint8)
    mask[:, : a[2].shape[1] // 2] = 1
    images = [Image(a[0]), Image(a[1]), Image(a[2], mask=mask), Image(b[0]), Image(b[1]), Image(np.zeros((480, 640), np.uint8))]
    intr = {i: (0.9 * im.value_array.shape[1], im.value_array.shape[1] / 2.0, im.value_array.shape[0] / 2.0) for i, im in enumerate(images)}
    return images, intr


def _config(detector):
    """-> (generator, detector plugin, matcher plugin)."""
    if detector == "superpoint":
        sp, sg = syn.superpoint_state_dict(0), syn.superglue_state_dict(1, "sharp")
        return (B200CorrespondenceGenerator(sp, max_keypoints=K, detector="superpoint", matcher="superglue", superglue_weights=sg),
                B200SuperPointDetectorDescriptor(max_keypoints=K, weights_path=sp), B200SuperGlueMatcher(weights_path=sg))
    if detector == "d2net":
        d2 = syn.d2net_state_dict(7)
        plugin = B200D2NetDetectorDescriptor(max_keypoints=K, model_path=d2)
        return B200CorrespondenceGenerator(max_keypoints=K, detector="d2net", matcher="twoway", d2net_weights=d2,
                                           ratio_test_threshold=RATIO), plugin, B200TwoWayMatcher(ratio_test_threshold=RATIO)
    plugin = (B200SIFTDetectorDescriptor if detector == "sift" else B200ORBDetectorDescriptor)(max_keypoints=K)
    return (B200CorrespondenceGenerator(max_keypoints=K, detector=detector, matcher="twoway", ratio_test_threshold=RATIO), plugin,
            B200TwoWayMatcher(ratio_test_threshold=RATIO))


def _rows(kp: Keypoints, desc: np.ndarray) -> np.ndarray:
    """One row per keypoint (x, y, scale, response, descriptor), sorted: the keypoint set independent of its order."""
    cols = [np.asarray(kp.coordinates, np.float64)]
    for f in (kp.scales, kp.responses):
        if f is not None:
            cols.append(np.asarray(f, np.float64)[:, None])
    d = np.asarray(desc, np.float64)
    m = np.concatenate(cols + [d.reshape(len(kp), d.shape[-1])], 1)
    return m[np.lexsort(m.T[::-1])] if len(m) else m


@pytest.mark.parametrize("detector", ["sift", "orb", "d2net", "superpoint"])
def test_generator_equals_plugins(golden_dir, detector):
    images, intr = _job(golden_dir)
    gen, det, mat = _config(detector)
    kps, matches = gen.generate_correspondences(None, images, PAIRS, verify_with=(intr, 4.0))
    feats = gen.last_device_features

    # keypoints and descriptors: the plugin's, as sets; the same Keypoints fields and dtypes
    for i, im in enumerate(images):
        pk, pd = det.detect_and_describe(im)
        gk, f = kps[i], feats[i]
        for field in ("coordinates", "scales", "responses"):
            a, b = getattr(gk, field), getattr(pk, field)
            assert (a is None) == (b is None) and (a is None or a.dtype == b.dtype), (detector, i, field)
        assert len(gk) == len(pk) == len(f) and f.desc.shape[1] == pd.shape[1], (detector, i)
        gd = f.desc.cpu().numpy()
        if detector == "sift":
            assert gd.dtype == np.uint8 and pd.dtype == np.float32  # the plugin's float32 copy of the uint8 descriptors
        if detector == "superpoint" and i == 5:
            continue  # the seeded network's scores on the flat image tie at the top-k boundary: the device keeps lower indices
        if detector == "superpoint":  # the device describe and the host describe agree to fp32 rounding
            g, p = _rows(gk, np.zeros((len(gk), 0))), _rows(pk, np.zeros((len(pk), 0)))
            assert np.array_equal(g, p), (detector, i)
            og = np.lexsort(np.asarray(gk.coordinates).T[::-1])
            op = np.lexsort(np.asarray(pk.coordinates).T[::-1])
            np.testing.assert_allclose(gd[og], pd[op], atol=1e-6)
        else:
            assert gd.dtype == (np.float32 if detector == "d2net" else np.uint8)
            assert np.array_equal(_rows(gk, gd), _rows(pk, pd)), (detector, i)
    flat_empty = detector in ("sift", "orb")  # the seeded D2-Net and SuperPoint networks still fire on the flat image
    assert len(kps[5]) == 0 or not flat_empty
    assert sum(len(k) for k in kps) > 2000

    # matches: the plugin's rows on the generator's own features, bit for bit, in the plugin's dtype
    assert sorted(matches) == sorted(PAIRS)
    for (i1, i2), m in matches.items():
        d1, d2 = feats[i1].desc.cpu().numpy(), feats[i2].desc.cpu().numpy()
        ref = mat.match(kps[i1], kps[i2], d1, d2, images[i1].value_array.shape, images[i2].value_array.shape)
        assert m.dtype == ref.dtype and np.array_equal(m, ref), (detector, i1, i2)
    assert sum(len(m) for m in matches.values()) > (0 if detector == "superpoint" else 100)  # SuperPoint / SuperGlue: seeded weights
    if flat_empty:
        assert len(matches[(4, 5)]) == 0 and len(matches[(0, 5)]) == 0

    # verification: B200Ransac.verify_many on the same keypoints (the float32 device coordinates) and rows
    ver = B200Ransac(True, 4.0)
    items = [(Keypoints(feats[i1].kp.cpu().numpy()), Keypoints(feats[i2].kp.cpu().numpy()), matches[(i1, i2)],
              Cal3Bundler(intr[i1][0], 0.0, 0.0, intr[i1][1], intr[i1][2]), Cal3Bundler(intr[i2][0], 0.0, 0.0, intr[i2][1], intr[i2][2]))
             for i1, i2 in PAIRS]
    verified = 0
    for p, (R, U, rows, ratio) in zip(PAIRS, ver.verify_many(items)):
        r = gen.last_two_view[p]
        assert (r.i2Ri1 is None) == (R is None), (detector, p)
        assert np.array_equal(r.v_corr_idxs.reshape(-1, 2), np.asarray(rows).reshape(-1, 2)) and r.inlier_ratio_est_model == ratio, (detector, p)
        if R is not None:
            verified += 1
            assert np.array_equal(r.i2Ri1.matrix(), R.matrix()) and np.array_equal(r.i2Ui1.point3(), U.point3()), (detector, p)
    assert verified >= 1, (detector, verified)
    if flat_empty:
        assert gen.last_two_view[(4, 5)].i2Ri1 is None and len(gen.last_two_view[(4, 5)].v_corr_idxs) == 0


def test_masked_images_give_the_plugin_masked_keypoints(golden_dir):
    """A SIFT and an ORB image with a mask (applied inside the batched device call) keep exactly the plugin's masked set, and
    none in the half the mask removes, which the same image without its mask has."""
    images, _ = _job(golden_dir)
    for detector in ("sift", "orb"):
        gen, det, _ = _config(detector)
        kps, _ = gen.generate_correspondences(None, [images[2], Image(images[2].value_array)], [(0, 1)])
        pk, pd = det.detect_and_describe(images[2])
        assert np.array_equal(_rows(kps[0], gen.last_device_features[0].desc.cpu().numpy()), _rows(pk, pd)), detector
        half = images[2].value_array.shape[1] / 2 + 1
        assert len(kps[0]) > 0 and np.all(np.asarray(kps[0].coordinates)[:, 0] < half)
        assert np.any(np.asarray(kps[1].coordinates)[:, 0] > half)
