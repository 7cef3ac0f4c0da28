"""GPU: the device-resident batched path (DeviceFrontEnd / B200CorrespondenceGenerator) agrees with the per-call plugins."""
import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib, synthetic as syn
from gtsfm_b200.correspondence_generator import B200CorrespondenceGenerator
from gtsfm_b200.detector_descriptor import SuperPointEngine
from gtsfm_b200.gtsfm_api import Image
from gtsfm_b200.matcher import LightGlueEngine
from gtsfm_b200.pipeline import DeviceFrontEnd
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu


def test_device_path_equals_host_path(b200_ctx):
    sp_sd, lg_sd = syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp")
    frames, cal = syn.synthetic_sequence(3, 240, 320)
    fe = DeviceFrontEnd(sp_sd, lg_sd, max_keypoints=600, ctx=b200_ctx)
    fa = fe.detect(torch.from_numpy(frames[0]).cuda())
    fb = fe.detect(torch.from_numpy(frames[2]).cuda())
    sp = SuperPointEngine(sp_sd, ctx=b200_ctx)
    xy, sc = sp.detect(frames[0])
    # device top-k = the 600 largest scores, kept in row-major order
    order = np.argsort(-sc, kind="stable")[:600]
    assert len(fa) == 600 and np.array_equal(fa.kp.cpu().numpy(), xy[np.sort(order)])
    np.testing.assert_allclose(fa.desc.cpu().numpy(), sp.describe(fa.kp.cpu().numpy()), atol=1e-6)
    m, stop = fe.match(fa, fb)
    lg = LightGlueEngine(lg_sd, ctx=b200_ctx)
    mh = lg.match(fa.kp.cpu().numpy(), fa.desc.cpu().numpy(), fb.kp.cpu().numpy(), fb.desc.cpu().numpy())
    assert np.array_equal(m.cpu().numpy(), mh) and len(mh) > 50
    E, R, t, ninl, mask = fe.verify(fa, fb, m, cal, cal, 4.0)
    assert E is not None and ninl > 0.8 * len(mh) and int(mask.sum().item()) == ninl
    n1 = vr.calibrate(fa.kp.cpu().numpy()[mh[:, 0]], *cal)
    n2 = vr.calibrate(fb.kp.cpu().numpy()[mh[:, 1]], *cal)
    assert np.array_equal(mask.cpu().numpy().astype(bool), vr.sampson_sq(E, n1, n2) < (4.0 / cal[0]) ** 2)
    assert abs(np.linalg.det(R) - 1) < 1e-6 and abs(np.linalg.norm(t) - 1) < 1e-6


def test_correspondence_generator_contract():
    sp_sd, lg_sd = syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp")
    frames, _ = syn.synthetic_sequence(4, 240, 320)
    gen = B200CorrespondenceGenerator(sp_sd, lg_sd, max_keypoints=500)
    graph = [(0, 1), (0, 2), (1, 3)]
    kps, matches = gen.generate_correspondences(None, [Image(f) for f in frames], graph)
    assert len(kps) == 4 and all(len(k) <= 500 and k.responses is not None for k in kps)
    assert sorted(matches) == sorted(graph)
    for (i1, i2), m in matches.items():
        assert m.dtype == np.int64 and m.shape[1] == 2 and len(m) > 20
        assert m[:, 0].max() < len(kps[i1]) and m[:, 1].max() < len(kps[i2])


def test_batched_match_equals_per_pair_and_golden(b200_ctx, golden_dir):
    """b2_lightglue_match_batched_dev: 11 ragged pairs (> one batch of 8; different sizes, early exit, pruning, empty
    image) walked in lock-step give exactly the rows of the per-pair entry point and of the reference fixtures."""
    from gtsfm_b200.pipeline import DeviceFeatures

    def feats(kp, sc, d, shape=(480, 640)):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        return DeviceFeatures(t(kp), t(sc), t(d), shape)

    for profile, cases in (("stop", [(8, 512, 512), (10, 2048, 1900), (21, 200, 180), (22, 300, 0), (23, 64, 700), (24, 1500, 1400),
                                      (25, 900, 901), (26, 333, 444), (27, 128, 128), (28, 1000, 256), (29, 50, 40)]),
                           ("prune", [(7, 700, 640), (9, 37, 5), (31, 800, 800)])):
        fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, profile), ctx=b200_ctx)
        pairs = []
        for seed, n0, n1 in cases:
            kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(seed, max(n0, 1), max(n1, 1))
            pairs.append((feats(kp0[:n0], sc0[:n0], d0[:n0]), feats(kp1[:n1], sc1[:n1], d1[:n1])))
        batched = fe.match_batch(pairs)
        stops = set()
        for (a, b), (mb, sb), (seed, n0, n1) in zip(pairs, batched, cases):
            ms, ss = fe.match(a, b)
            assert sb == ss and np.array_equal(mb.cpu().numpy(), ms.cpu().numpy()), (profile, seed, n0, n1)
            stops.add(sb)
            tag = golden_dir / f"lightglue_{profile}_{seed}.npz"
            if tag.exists():
                fx = np.load(tag)
                assert sb == int(fx["stop"]) and np.array_equal(mb.cpu().numpy(), fx["matches"])
        assert len(stops) >= 2 or profile == "prune", "the batch should mix stopping layers"


def test_detect_many_equals_detect(b200_ctx):
    """The no-sync multi-image path (b2_superpoint_extract_async_dev) gives the same features as one synchronous detect per
    image, on mixed image sizes and a flat image.  The SuperPoint network has one launch path: there is no graph option."""
    sp_sd = syn.superpoint_state_dict(0)
    frames, _ = syn.synthetic_sequence(4, 240, 320)
    big, _ = syn.synthetic_sequence(2, 480, 640)
    imgs = [torch.from_numpy(f).cuda() for f in (frames[0], big[0], frames[1], big[1], frames[2])]
    imgs.append(torch.zeros((240, 320), dtype=torch.uint8, device="cuda"))  # flat image
    fe = DeviceFrontEnd(sp_sd, None, max_keypoints=700, ctx=b200_ctx)
    ref = [fe.detect(im) for im in imgs]
    assert len(ref[1]) == 700 and 0 < len(ref[0]) <= 700
    many = fe.detect_many(imgs)
    for r, got in zip(ref, many):
        assert len(got) == len(r) and got.shape == r.shape
        assert torch.equal(got.kp, r.kp) and torch.equal(got.score, r.score) and torch.equal(got.desc, r.desc)
    with pytest.raises(_lib.B200Error, match="unknown option"):
        b200_ctx.set_option("superpoint_graph", 1)


def test_superglue_lanes_and_lightglue_batches_equal_sequential(b200_ctx, monkeypatch):
    """match_superglue_many with several library contexts on several streams returns what the single-lane calls do, and
    match_many's lock-step batches return what one pair per batch does."""
    from gtsfm_b200 import pipeline

    sp_sd, lg_sd, sg_sd = syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), syn.superglue_state_dict(1, "sharp")
    frames, _ = syn.synthetic_sequence(5, 240, 320)
    fe = DeviceFrontEnd(sp_sd, lg_sd, max_keypoints=500, ctx=b200_ctx, superglue_sd=sg_sd)
    feats = fe.detect_many([torch.from_numpy(f).cuda() for f in frames])
    pairs = [(feats[i], feats[j]) for i in range(5) for j in range(i + 1, 5)] * 2  # 20 pairs = 3 lock-step batches
    ref_lg = [fe.match_batch([p])[0] for p in pairs[:10]]
    ref_sg = [fe.match_superglue(*p) for p in pairs[:10]]
    monkeypatch.setattr(pipeline, "SG_LANES", 3)
    seen = []
    got_lg = fe.match_many(pairs, on_chunk=lambda c0, res: seen.append((c0, len(res))))
    got_sg = fe.match_superglue_many(pairs)
    assert sorted(seen) == [(0, 8), (8, 8), (16, 4)] and len(fe._lanes["superglue"]) == 3
    for i in range(20):
        assert torch.equal(got_lg[i][0], ref_lg[i % 10][0]) and got_lg[i][1] == ref_lg[i % 10][1]
        assert torch.equal(got_sg[i], ref_sg[i % 10])
    assert sum(int(m.shape[0]) for m, _ in got_lg) > 200
