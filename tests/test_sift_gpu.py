"""GPU suite of the SIFT detector-descriptor (csrc/sift.cu): parity with cv2 against the goldens written by the reference's
unmodified SIFTDetectorDescriptor (oracle/make_golden_sift.py), and the properties that hold exactly: order, de-duplication,
the mask rule, run-to-run and batched-versus-single results, input layouts, top-k selections and the matcher hand-off."""
import numpy as np
import pytest

from oracle import sift_ref, twoway_ref

pytestmark = pytest.mark.gpu

NONEMPTY = [c for c in sift_ref.CASES if c not in ("empty_8", "empty_16", "flat")]


def golden(golden_dir, name):
    f = np.load(golden_dir / f"sift_{name}.npz")
    return {k: f[k] for k in sift_ref.FIELDS}, f["desc"]


def rec(kp):
    return {f: np.asarray(kp[f]) for f in sift_ref.FIELDS}


def from_dev(kp, desc):
    """extract_many's (n, 6) float32 device records -> host structured records and descriptors."""
    from gtsfm_b200 import _lib

    return np.ascontiguousarray(kp.cpu().numpy()).view(_lib.SIFT_KEYPOINT_DTYPE).reshape(-1), desc.cpu().numpy()


@pytest.fixture(scope="module")
def eng(b200_ctx):
    from gtsfm_b200.detector_descriptor import SiftEngine

    return SiftEngine(ctx=b200_ctx)


@pytest.fixture(scope="module")
def lund_host(eng, golden_dir):
    return {i: eng.detect_and_describe(*sift_ref.case_image(f"lund_{i}", golden_dir)) for i in range(1, 6)}


@pytest.mark.parametrize("name", sift_ref.CASES)
def test_parity_with_cv2(eng, golden_dir, name):
    arr, mask = sift_ref.case_image(name, golden_dir)
    kp, desc = eng.detect_and_describe(arr, mask)
    ref, rdesc = golden(golden_dir, name)
    assert desc.dtype == np.uint8 and desc.shape == (len(kp), 128)
    if len(ref["x"]) == 0:
        assert len(kp) == 0
        return
    p = sift_ref.parity(rec(kp), desc, ref, rdesc)
    print(name, p)
    if name == "synthetic_12mp":
        # The byte cvRound((xi + 0.5) * 255) of the packed octave quantises the sub-layer offset xi; float noise of ~1e-4 in xi
        # moves it by one at rounding boundaries.  On this frame cv2's own scalar build corresponds to its default build at
        # 98.96 % under the full criterion (99.46 % on the lund frames), so the full criterion is held at 98.5 % here and the
        # 99 % bar applies with that byte left out.
        assert p["a_in_b"] >= 0.985 and p["b_in_a"] >= 0.985, p
        p = sift_ref.parity(rec(kp), desc, ref, rdesc, octave_bits=0xFFFF)
    assert p["a_in_b"] >= 0.99 and p["b_in_a"] >= 0.99, p
    assert abs(p["count_ratio"] - 1.0) <= 0.01, p
    assert p["desc_within_1"] >= 0.995, p


@pytest.mark.parametrize("name", ["lund_1", "odd_crop"])
def test_gaussian_pyramid_levels(b200_ctx, eng, golden_dir, name):
    arr, _ = sift_ref.case_image(name, golden_dir)
    eng.detect_and_describe(arr)
    ref = sift_ref.gaussian_pyramid(arr)
    total = sum(lv.size for o in ref for lv in o)
    got = b200_ctx.debug_fetch("sift_pyramid", total)
    assert got.size == total
    off = 0
    for o, levels in enumerate(ref):
        for i, lv in enumerate(levels):
            g = got[off: off + lv.size].reshape(lv.shape)
            off += lv.size
            assert np.abs(g - lv).max() <= 1e-3, (o, i, np.abs(g - lv).max())


def test_order_and_deduplication(lund_host):
    for kp, _ in lund_host.values():
        assert np.array_equal(np.lexsort((kp["angle"], -kp["size"], kp["y"], kp["x"])), np.arange(len(kp)))
        same = ((kp["x"][1:] == kp["x"][:-1]) & (kp["y"][1:] == kp["y"][:-1]) & (kp["size"][1:] == kp["size"][:-1])
                & (kp["angle"][1:] == kp["angle"][:-1]))
        assert not same.any()


def test_mask_rule_is_exact(eng, golden_dir):
    arr, mask = sift_ref.case_image("lund_2_mask", golden_dir)
    full, fd = eng.detect_and_describe(arr)
    kp, desc = eng.detect_and_describe(arr, mask)
    keep = mask[(full["y"] + np.float32(0.5)).astype(np.int32), (full["x"] + np.float32(0.5)).astype(np.int32)] != 0
    assert np.array_equal(kp, full[keep]) and np.array_equal(desc, fd[keep])
    none, nd = eng.detect_and_describe(arr, np.zeros_like(mask))
    assert len(none) == 0 and nd.shape == (0, 128)


def test_run_to_run_and_batched_equal_single(eng, golden_dir, lund_host):
    import torch

    again = eng.detect_and_describe(*sift_ref.case_image("lund_3", golden_dir))
    assert np.array_equal(again[0], lund_host[3][0]) and np.array_equal(again[1], lund_host[3][1])
    imgs = [torch.from_numpy(sift_ref.case_image(f"lund_{i}", golden_dir)[0]).cuda() for i in range(1, 6)]
    for _ in range(2):
        out = eng.extract_many(imgs, max_keypoints=100000)
        for i, (kp, desc, total) in zip(range(1, 6), out):
            k, d = from_dev(kp, desc)
            assert total == len(lund_host[i][0])
            assert np.array_equal(k, lund_host[i][0]) and np.array_equal(d, lund_host[i][1])


def test_gray_rgb_rgba_and_pitched_input_agree(eng, golden_dir, lund_host):
    import torch

    g, _ = sift_ref.case_image("lund_4", golden_dir)
    base = lund_host[4]
    for arr in (np.repeat(g[..., None], 3, 2), np.concatenate([np.repeat(g[..., None], 3, 2), np.full_like(g, 9)[..., None]], 2)):
        kp, desc = eng.detect_and_describe(arr)
        assert np.array_equal(kp, base[0]) and np.array_equal(desc, base[1])
    rgb, _ = sift_ref.case_image("lund_4_rgb", golden_dir)
    kp, desc = eng.detect_and_describe(sift_ref.rgb_to_gray_cv(rgb))
    kp2, desc2 = eng.detect_and_describe(rgb)
    assert np.array_equal(kp, kp2) and np.array_equal(desc, desc2)
    wide = torch.zeros((g.shape[0], g.shape[1] + 72), dtype=torch.uint8, device="cuda")
    wide[:, 40: 40 + g.shape[1]] = torch.from_numpy(g).cuda()
    (k, d, _), = eng.extract_many([wide[:, 40: 40 + g.shape[1]]], max_keypoints=100000)
    k, d = from_dev(k, d)
    assert np.array_equal(k, base[0]) and np.array_equal(d, base[1])


def test_device_topk_equals_numpy_selection(eng, golden_dir, lund_host):
    import torch

    imgs = [torch.from_numpy(sift_ref.case_image(f"lund_{i}", golden_dir)[0]).cuda() for i in (1, 2)]
    for k in (1, 1000, 5000):
        for i, (kp, desc, total) in zip((1, 2), eng.extract_many(imgs, max_keypoints=k)):
            full, fd = lund_host[i]
            sel = np.sort(np.argsort(-full["response"], kind="stable")[:k])
            got, gd = from_dev(kp, desc)
            assert total == len(full) and np.array_equal(got, full[sel]) and np.array_equal(gd, fd[sel])


def test_plugin_selection_is_the_reference_argpartition(golden_dir, lund_host):
    from gtsfm_b200.detector_descriptor import B200SIFTDetectorDescriptor
    from gtsfm_b200.gtsfm_api import Image

    full, fd = lund_host[1]
    det = B200SIFTDetectorDescriptor(max_keypoints=5000)
    kps, desc = det.detect_and_describe(Image(sift_ref.case_image("lund_1", golden_dir)[0]))
    sel = np.argpartition(-full["response"].astype(np.float64), 5000)[:5000]
    assert np.array_equal(kps.coordinates, np.stack([full["x"], full["y"]], 1).astype(np.float64)[sel])
    assert np.array_equal(kps.scales, full["size"].astype(np.float64)[sel])
    assert np.array_equal(kps.responses, full["response"].astype(np.float64)[sel])
    assert desc.dtype == np.float32 and np.array_equal(desc, fd[sel].astype(np.float32))


def test_device_descriptors_into_device_matcher_are_exact(b200_ctx, eng, golden_dir):
    import torch

    from gtsfm_b200.matcher import TwoWayEngine

    imgs = [torch.from_numpy(sift_ref.case_image(f"lund_{i}", golden_dir)[0]).cuda() for i in (1, 2, 3)]
    out = eng.extract_many(imgs, max_keypoints=5000)
    pairs = [(out[0][1], out[1][1]), (out[1][1], out[2][1])]
    res = TwoWayEngine(ctx=b200_ctx).match_batched_dev(pairs, 0.8)
    for (a, b), m in zip(pairs, res):
        ref, _ = twoway_ref.twoway_match(a.cpu().numpy().astype(np.float32), b.cpu().numpy().astype(np.float32), 0.8)
        assert np.array_equal(m.cpu().numpy(), ref.astype(np.int64)) and len(ref) > 100


@pytest.mark.parametrize("i", [1, 2, 3, 4])
def test_matches_agree_with_cv2_sift_matches(b200_ctx, golden_dir, lund_host, i):
    from gtsfm_b200.matcher import TwoWayEngine

    mt = TwoWayEngine(ctx=b200_ctx)
    (ka, da), (kb, db) = lund_host[i], lund_host[i + 1]
    ra, rda = golden(golden_dir, f"lund_{i}")
    rb, rdb = golden(golden_dir, f"lund_{i + 1}")
    ref, _ = twoway_ref.twoway_match(rda.astype(np.float32), rdb.astype(np.float32), 0.8)
    got = mt.match(da, db, 0.8)
    ia, ja = sift_ref.correspond(rec(ka), ra)
    ib, jb = sift_ref.correspond(rec(kb), rb)
    ma, mb = dict(zip(ia.tolist(), ja.tolist())), dict(zip(ib.tolist(), jb.tolist()))
    ref_set = set(map(tuple, ref.astype(np.int64).tolist()))
    agree = sum((ma.get(x), mb.get(y)) in ref_set for x, y in got.tolist())
    assert agree / len(got) >= 0.98, (agree, len(got), len(ref))
    assert abs(len(got) / len(ref) - 1.0) <= 0.01, (len(got), len(ref))


def test_edge_cases(eng, golden_dir):
    from gtsfm_b200 import _lib
    from gtsfm_b200.detector_descriptor import B200SIFTDetectorDescriptor
    from gtsfm_b200.gtsfm_api import Image

    det = B200SIFTDetectorDescriptor()
    for name in ("empty_8", "empty_16", "flat"):
        kps, desc = det.detect_and_describe(Image(sift_ref.case_image(name, golden_dir)[0]))
        assert len(kps) == 0 and desc.shape == (0, 128) and desc.dtype == np.float32
    kps, desc = det.detect_and_describe(Image(sift_ref.case_image("tiny_crop", golden_dir)[0]))
    assert len(kps) == 2 and desc.shape == (2, 128)
    with pytest.raises(_lib.B200Error):
        eng.detect_and_describe(np.zeros((4100, 4100), np.uint8))
    with pytest.raises(ValueError):
        det.detect_and_describe(Image(np.zeros((64, 64, 2), np.uint8)))


def test_host_entry_retries_when_capacity_is_short(b200_ctx, golden_dir, lund_host):
    from gtsfm_b200.detector_descriptor import SiftEngine

    small = SiftEngine(ctx=b200_ctx, capacity=1)
    kp, desc = small.detect_and_describe(sift_ref.case_image("lund_5", golden_dir)[0])
    assert small.capacity == len(kp) and np.array_equal(kp, lund_host[5][0]) and np.array_equal(desc, lund_host[5][1])
