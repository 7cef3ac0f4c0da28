"""GPU parity on BASELINE configs[0]: all 12 lund-door images and the 66 exhaustive pairs (deep_front_end.yaml: SuperPoint, max 5000
keypoints, LightGlue) against what the UNMODIFIED reference modules produced (oracle/make_golden.py::golden_lund_door).

Keypoints / scores are compared for every detection; the reference's own top-k SELECTION is then fed to describe + match, so
that the argpartition tie at the k-th score (tests/test_lightglue_gpu.py::test_lund_pair_and_crop_chain documents it) cannot
renumber rows: match indices must be bit-identical for all 66 pairs.  The top-k boundary itself is tested separately."""
import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.detector_descriptor import SuperPointEngine
from gtsfm_b200.matcher import LightGlueEngine

pytestmark = pytest.mark.gpu

_cache = {}


def _features(b200_ctx, golden_dir):
    """detect all 12 frames once; describe at the reference-selected keypoints."""
    if "feats" in _cache:
        return _cache["img"], _cache["feats"]
    img = np.load(golden_dir / "lund_door_images.npz")
    sp = SuperPointEngine(syn.superpoint_state_dict(0), ctx=b200_ctx)
    feats = {}
    for i in range(1, 13):
        xy, sc = sp.detect(img[f"gray_{i}"])
        sel = img[f"sel_{i}"]
        ref_xy = img[f"kp_{i}"].astype(np.float32)
        desc = sp.describe(ref_xy[sel])
        feats[i] = dict(xy=xy, sc=sc, sel_xy=ref_xy[sel], desc=desc)
    _cache["img"], _cache["feats"] = img, feats
    return img, feats


@pytest.mark.parametrize("i", range(1, 13))
def test_detection_equals_reference(b200_ctx, golden_dir, i):
    img, feats = _features(b200_ctx, golden_dir)
    f = feats[i]
    ref_xy = img[f"kp_{i}"].astype(np.float32)
    assert f["xy"].shape == ref_xy.shape, f"image {i}: {len(f['xy'])} keypoints vs reference {len(ref_xy)}"
    if not np.array_equal(f["xy"], ref_xy):
        # simple_nms compares floats with == (superpoint.py:51-61): two neighbouring pixels whose scores differ by an ulp
        # in the reference's MKL-DNN arithmetic can tie - or order the other way - in ours, and the surviving pixel of that
        # 9 x 9 window moves (and with it, through the suppression rounds, possibly its neighbour).  Allowed: at most two
        # moved keypoints per image, each within the NMS radius of the reference's.
        mine, ref = set(map(tuple, f["xy"].tolist())), set(map(tuple, ref_xy.tolist()))
        only_m, only_r = sorted(mine - ref), sorted(ref - mine)
        _cache.setdefault("moved", []).append((i, only_m, only_r))
        assert len(only_m) == len(only_r) <= 2, f"image {i}: {len(only_m)} / {len(only_r)} keypoints differ: {only_m[:4]} vs {only_r[:4]}"
        for km in only_m:
            assert min(max(abs(km[0] - kr[0]), abs(km[1] - kr[1])) for kr in only_r) <= 4, (only_m, only_r)
        keep = np.array([tuple(k) in ref for k in f["xy"].tolist()])
        keep_r = np.array([tuple(k) in mine for k in ref_xy.tolist()])
        assert np.array_equal(f["xy"][keep], ref_xy[keep_r]), f"image {i}: order of the common keypoints differs"
        np.testing.assert_allclose(f["sc"][keep], img[f"sc_{i}"][keep_r], rtol=0, atol=1e-5)
        print(f"image {i}: NMS tie moved keypoints {only_r} -> {only_m}")
        return
    np.testing.assert_allclose(f["sc"], img[f"sc_{i}"], rtol=0, atol=1e-5)
    assert np.abs(f["desc"][::20] - img[f"desc_{i}"]).max() < 1e-3  # north_star: descriptors within 1e-3
    # top-k boundary: the GPU scores select the same 5000 keypoints up to swaps among scores within 1e-6 of the k-th
    sel_gpu = set(np.argpartition(-f["sc"], 5000)[:5000].tolist())
    sel_ref = set(img[f"sel_{i}"].tolist())
    kth = np.sort(img[f"sc_{i}"][img[f"sel_{i}"]])[0]
    odd = sel_gpu ^ sel_ref
    assert len(odd) <= 6 and all(abs(img[f"sc_{i}"][j] - kth) < 1e-6 for j in odd), (len(odd), kth)


def test_moved_keypoints_are_rare(b200_ctx, golden_dir):
    """Over the 207 000 detections of the 12 frames at most 3 may sit in a different pixel of their NMS window."""
    _features(b200_ctx, golden_dir)
    assert sum(len(m[1]) for m in _cache.get("moved", [])) <= 3, _cache.get("moved")


def test_all_66_pairs_bit_identical(b200_ctx, golden_dir):
    img, feats = _features(b200_ctx, golden_dir)
    fx = np.load(golden_dir / "lund_door_66pairs.npz")
    lg = LightGlueEngine(syn.lightglue_state_dict(2, str(fx["profile"])), ctx=b200_ctx)
    bad, total = [], 0
    for a in range(1, 13):
        for b in range(a + 1, 13):
            m = lg.match(feats[a]["sel_xy"], feats[a]["desc"], feats[b]["sel_xy"], feats[b]["desc"])
            ref = fx[f"m_{a}_{b}"].astype(np.int64)
            total += len(ref)
            if lg.last_stop != int(fx[f"stop_{a}_{b}"]) or not np.array_equal(m, ref):
                bad.append((a, b, len(m), len(ref), lg.last_stop))
    assert total > 4000
    assert not bad, f"{len(bad)} of 66 pairs differ from the reference: {bad[:8]}"
