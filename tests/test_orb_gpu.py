"""GPU suite of the ORB detector-descriptor (csrc/orb.cu): bit-exact parity with cv2 against the goldens written by the
reference's unmodified ORBDetectorDescriptor (oracle/make_golden_orb.py), every stage against oracle/orb_ref.py, the output
order, batched-versus-single and run-to-run results, input layouts, the mask rule, the capacity contract and the hand-off to
the two-way matcher and the verifier."""
import ctypes as C

import numpy as np
import pytest

from oracle import orb_ref, twoway_ref

pytestmark = pytest.mark.gpu

OC_N, OC_SEL = 32, 8  # csrc/orb.cu's per-image counters: their number, the selection-1 counts per level


def golden(golden_dir, name):
    f = np.load(golden_dir / f"orb_{name}.npz")
    return {k: f[k] for k in orb_ref.FIELDS}, f["desc"]


def rec(kp):
    return {f: np.asarray(kp[f]) for f in orb_ref.FIELDS}


def assert_same(a, da, b, db):
    ia, ib = orb_ref.same_keypoints(a, da, b, db)
    for f in orb_ref.FIELDS:
        assert np.array_equal(np.asarray(a[f])[ia].view(np.int32), np.asarray(b[f])[ib].view(np.int32)), f
    assert np.array_equal(da[ia], db[ib])


def from_dev(kp, desc):
    from gtsfm_b200 import _lib

    return np.ascontiguousarray(kp.cpu().numpy()).view(_lib.SIFT_KEYPOINT_DTYPE).reshape(-1), desc.cpu().numpy()


def layout(h, w):
    """csrc/orb.cu's ob_geom: byte-plane offsets (16-byte padded levels) and candidate-list offsets."""
    sizes = orb_ref.level_sizes(h, w)
    off, coff, L, Cn = [], [], 0, 0
    for lh, lw in sizes:
        off.append(L)
        coff.append(Cn)
        L += (lh * lw + 15) // 16 * 16
        Cn += ((lw + 1) // 2) * ((lh + 1) // 2)
    return sizes, off, L, coff, Cn


@pytest.fixture(scope="module")
def eng(b200_ctx):
    from gtsfm_b200.detector_descriptor import OrbEngine

    return OrbEngine(ctx=b200_ctx)


@pytest.mark.parametrize("name", orb_ref.CASES)
def test_parity_with_cv2(eng, golden_dir, name):
    arr, mask = orb_ref.case_image(name, golden_dir)
    kp, desc = eng.detect_and_describe(arr, mask)
    ref, rdesc = golden(golden_dir, name)
    assert desc.dtype == np.uint8 and desc.shape == (len(kp), 32)
    assert_same(rec(kp), desc, ref, rdesc)


@pytest.mark.parametrize("name", ["lund_1", "lund_2_mask", "odd_crop", "synthetic_12mp"])
def test_output_order_and_restatement(eng, golden_dir, name):
    arr, mask = orb_ref.case_image(name, golden_dir)
    kp, desc = eng.detect_and_describe(arr, mask)
    r, d = orb_ref.orb(arr, mask)
    for f in orb_ref.FIELDS:  # orb_ref writes the documented order: level, response descending, y, x
        assert np.array_equal(np.asarray(kp[f]).view(np.int32), r[f].view(np.int32)), f
    assert np.array_equal(desc, d)


@pytest.mark.parametrize("name", ["lund_2_mask", "odd_crop", "low_levels"])
def test_stages_against_the_restatement(b200_ctx, eng, golden_dir, name):
    arr, mask = orb_ref.case_image(name, golden_dir)
    eng.detect_and_describe(arr, mask)
    st = {}
    orb_ref.orb(arr, mask, stages=st)
    sizes, off, L, coff, Cn = layout(*arr.shape[:2])
    planes = {k: b200_ctx.debug_fetch(f"orb_{k}", L // 4).view(np.uint8) for k in ("levels", "scores", "blurred", "masks")}
    counts = b200_ctx.debug_fetch("orb_counts", OC_N).view(np.int32)
    sel = b200_ctx.debug_fetch("orb_sel", Cn).view(np.int32)
    harris = b200_ctx.debug_fetch("orb_harris", Cn)
    mpyr = orb_ref.mask_pyramid(mask) if mask is not None else None
    for l, (h, w) in enumerate(sizes):
        for k, ref in (("levels", st["levels"][l]), ("scores", st["scores"][l]), ("blurred", st["blurred"][l])):
            assert np.array_equal(planes[k][off[l]: off[l] + h * w].reshape(h, w), ref), (k, l)
        if mpyr is not None:
            assert np.array_equal(planes["masks"][off[l]: off[l] + h * w].reshape(h, w), mpyr[l]), ("masks", l)
        y, x = st["cand"][l]
        m = counts[OC_SEL + l]
        assert m == len(y), l
        got = {int(v): float(r) for v, r in zip(sel[coff[l]: coff[l] + m], harris[coff[l]: coff[l] + m])}
        want = {int((a << 16) | b): float(r) for a, b, r in zip(y, x, st["harris"][l])}
        assert set(got) == set(want), l
        assert all(np.float32(got[k]).view(np.int32) == np.float32(want[k]).view(np.int32) for k in got), l


def test_batched_equals_single_and_run_to_run(eng, golden_dir):
    import torch

    imgs = [orb_ref.case_image(f"lund_{i}", golden_dir)[0] for i in range(1, 6)]
    dev = [torch.from_numpy(x).cuda() for x in imgs]
    a = eng.extract_many(dev)
    b = eng.extract_many(dev)
    for i, x in enumerate(dev):
        (s,) = eng.extract_many([x])
        for t in (b[i], s):
            assert torch.equal(a[i][0], t[0]) and torch.equal(a[i][1], t[1]) and a[i][2] == t[2]
        kp, desc = from_dev(a[i][0], a[i][1])
        hk, hd = eng.detect_and_describe(imgs[i])
        assert np.array_equal(kp.view(np.int32), hk.view(np.int32)) and np.array_equal(desc, hd)


def test_gray_rgb_rgba_and_pitched_input_agree(eng, golden_dir):
    import torch

    for name in ("lund_4_rgb", "lund_4_rgba"):
        arr, _ = orb_ref.case_image(name, golden_dir)
        gray = orb_ref.rgb_to_gray_cv(arr)
        hk, hd = eng.detect_and_describe(gray)
        wide = torch.zeros((arr.shape[0], arr.shape[1] + 13, arr.shape[2]), dtype=torch.uint8, device="cuda")
        wide[:, : arr.shape[1]] = torch.from_numpy(arr).cuda()
        pitched = wide[:, : arr.shape[1]]
        assert pitched.stride(0) != arr.shape[1] * arr.shape[2]
        (got,) = eng.extract_many([pitched])
        kp, desc = from_dev(got[0], got[1])
        assert np.array_equal(kp.view(np.int32), hk.view(np.int32)) and np.array_equal(desc, hd)


def test_mask_rule_on_the_batched_path(eng, golden_dir):
    import torch

    arr, mask = orb_ref.case_image("lund_2_mask", golden_dir)
    ref, rdesc = golden(golden_dir, "lund_2_mask")
    (got,) = eng.extract_many([torch.from_numpy(arr).cuda()], [torch.from_numpy(mask * 255).cuda()])
    kp, desc = from_dev(got[0], got[1])
    assert_same(rec(kp), desc, ref, rdesc)


def test_top_k_on_the_batched_path(eng, golden_dir):
    import torch

    arr, _ = orb_ref.case_image("lund_3", golden_dir)
    hk, hd = eng.detect_and_describe(arr)
    (got,) = eng.extract_many([torch.from_numpy(arr).cuda()], max_keypoints=77)
    kp, desc = from_dev(got[0], got[1])
    assert got[2] == len(hk) and len(kp) == 77
    keep = np.sort(np.argsort(-hk["response"].astype(np.float64), kind="stable")[:77])
    assert np.array_equal(kp.view(np.int32), hk[keep].view(np.int32)) and np.array_equal(desc, hd[keep])


def test_capacity_contract(b200_ctx, golden_dir):
    from gtsfm_b200 import _lib

    arr, _ = orb_ref.case_image("lund_1", golden_dir)
    kp = np.empty(10, _lib.SIFT_KEYPOINT_DTYPE)
    desc = np.empty((10, 32), np.uint8)
    n = C.c_int(0)
    rc = b200_ctx.lib.b2_orb_detect_host(b200_ctx.handle, _lib.ptr(arr), arr.shape[0], arr.shape[1], 1, None, _lib.ptr(kp),
                                         _lib.ptr(desc), 10, C.byref(n))
    assert rc == _lib.SIFT_CAPACITY and n.value == 500


def test_plugin_matches_reference_plugin(golden_dir):
    from gtsfm_b200.detector_descriptor import B200ORBDetectorDescriptor
    from gtsfm_b200.gtsfm_api import Image

    p = B200ORBDetectorDescriptor(max_keypoints=120)
    for name in ("lund_2_mask", "flat"):
        arr, mask = orb_ref.case_image(name, golden_dir)
        kp, desc = p.detect_and_describe(Image(arr, mask=mask))
        c, s, r, d = orb_ref.detect_and_describe(arr, mask, max_keypoints=120)
        assert desc.dtype == np.uint8 and desc.shape == (len(c), 32)
        key = lambda cc, dd: sorted(zip(map(tuple, cc), map(bytes, dd)))  # noqa: E731
        assert key(kp.coordinates, desc) == key(c, d)


def test_front_end_match_and_verify(eng, golden_dir):
    """Device ORB -> b2_mnn_match_batched_dev (u8, dim 32) at ratio 0.8 on lund (1, 2) .. (4, 5): equal to the reference's
    TwoWayMatcher on the same descriptors; once permuted into cv2's keypoint order, equal to the reference's ORB + TwoWayMatcher;
    and B200Ransac verifies the matches."""
    import torch

    from gtsfm_b200.gtsfm_api import Cal3Bundler, Keypoints
    from gtsfm_b200.matcher import TwoWayEngine
    from gtsfm_b200.verifier import B200Ransac

    imgs = [orb_ref.case_image(f"lund_{i}", golden_dir)[0] for i in range(1, 6)]
    feats = eng.extract_many([torch.from_numpy(x).cuda() for x in imgs])
    pairs = [(feats[i][1], feats[i + 1][1]) for i in range(4)]
    got = TwoWayEngine(ctx=eng.ctx).match_batched_dev(pairs, ratio=0.8)
    host = [from_dev(kp, d) for kp, d, _ in feats]
    gold = [golden(golden_dir, f"lund_{i}") for i in range(1, 6)]
    ver = B200Ransac(use_intrinsics_in_verification=False, estimation_threshold_px=4.0)
    cal = Cal3Bundler(1000.0, 0.0, 0.0, 380.0, 567.0)
    for i in range(4):
        m = got[i].cpu().numpy()
        ref, _ = twoway_ref.twoway_match(host[i][1], host[i + 1][1], 0.8)
        assert np.array_equal(m, ref.astype(np.int64).reshape(-1, 2)), i
        # into cv2's order: perm[k] = the device index of cv2's keypoint k
        perms = []
        for j in (i, i + 1):
            ia, ib = orb_ref.same_keypoints(rec(host[j][0]), host[j][1], gold[j][0], gold[j][1])
            perm = np.empty(len(ia), np.int64)
            perm[ib] = ia
            perms.append(perm)
        ref_cv2, _ = twoway_ref.twoway_match(gold[i][1], gold[i + 1][1], 0.8)
        ref_cv2 = ref_cv2.astype(np.int64).reshape(-1, 2)
        mine_cv2, _ = twoway_ref.twoway_match(host[i][1][perms[0]], host[i + 1][1][perms[1]], 0.8)
        assert np.array_equal(mine_cv2.astype(np.int64).reshape(-1, 2), ref_cv2), i
        raw = set(zip(perms[0][ref_cv2[:, 0]], perms[1][ref_cv2[:, 1]]))
        agree = len(raw & set(map(tuple, m))) / max(len(raw), 1)
        assert agree >= 0.98, (i, agree)
        kp1 = Keypoints(np.stack([host[i][0]["x"], host[i][0]["y"]], 1).astype(np.float64))
        kp2 = Keypoints(np.stack([host[i + 1][0]["x"], host[i + 1][0]["y"]], 1).astype(np.float64))
        R, t, inl, ratio = ver.verify(kp1, kp2, m, cal, cal)
        assert R is not None and len(inl) > 0 and 0 < ratio <= 1, i
