"""GPU: LightGlue pairs that start from per-image encodings (b2_lightglue_encode_batched_dev: the state after layer 0's self
block, made once per image) match exactly as pairs that start from the features."""
import ctypes as C

import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn
from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd

pytestmark = pytest.mark.gpu


def _feats(kp, sc, d):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return DeviceFeatures(t(kp), t(sc), t(d), (480, 640))


def _images():
    """Ragged images (one empty) and pairs over them: images in several pairs of one batch, 10 pairs = two batches."""
    ims = []
    for seed, n0, n1 in ((8, 512, 512), (10, 1900, 1700), (21, 200, 180), (24, 1500, 1400), (29, 50, 40)):
        kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(seed, n0, n1)
        ims += [_feats(kp0, sc0, d0), _feats(kp1, sc1, d1)]
    ims.append(_feats(np.zeros((0, 2), np.float32), np.zeros(0, np.float32), np.zeros((0, 256), np.float32)))
    idx = [(0, 1), (2, 3), (0, 3), (4, 5), (10, 1), (6, 7), (2, 1), (8, 9), (0, 10), (6, 3)]
    return ims, [(ims[i], ims[j]) for i, j in idx]


def _run(fe, pairs, use_enc, key=None):
    """b2_lightglue_match_batched_dev with scores; use_enc[i] = (enc0?, enc1?) -> [(rows, scores, stop)]."""
    n = len(pairs)
    arr = (_lib.LightGluePair * n)()
    outs = []
    for i, (a, b) in enumerate(pairs):
        cap = max(1, min(len(a), len(b)))
        m = torch.empty((cap, 2), dtype=torch.int64, device="cuda")
        s = torch.empty(cap, dtype=torch.float32, device="cuda")
        outs.append((m, s))
        arr[i].kp0, arr[i].desc0, arr[i].n0 = a.kp.data_ptr(), a.desc.data_ptr(), len(a)
        arr[i].kp1, arr[i].desc1, arr[i].n1 = b.kp.data_ptr(), b.desc.data_ptr(), len(b)
        arr[i].enc0 = a.enc[key].data_ptr() if use_enc[i][0] else None
        arr[i].enc1 = b.enc[key].data_ptr() if use_enc[i][1] else None
        arr[i].out_matches, arr[i].out_scores = m.data_ptr(), s.data_ptr()
    prm = _lib.LightGlueParams(0.95, 0.99, 0.1, fe.prune_min, fe.fp16_attention)
    fe.ctx.check(fe.lib.b2_lightglue_match_batched_dev(fe.ctx.handle, arr, n, C.byref(prm), fe._stream()), "match_batched_dev")
    return [(m[: arr[i].out_k].cpu().numpy(), s[: arr[i].out_k].cpu().numpy(), int(arr[i].out_stop_layer)) for i, (m, s) in enumerate(outs)]


def _check_encoded_equals_plain(fe, score_atol=2e-4):
    ims, pairs = _images()
    plain = _run(fe, pairs, [(False, False)] * len(pairs))
    key = fe.encode(ims)
    assert all(key in f.enc for f in ims)
    full = _run(fe, pairs, [(True, True)] * len(pairs), key)
    mixed = _run(fe, pairs, [(i % 2 == 0, i % 3 == 0) for i in range(len(pairs))], key)
    batched = fe.match_batch(pairs)
    for (a, b), p, e, x, (mb, sb) in zip(pairs, plain, full, mixed, batched):
        ms, ss = fe.match(a, b)
        for got in (e, x):
            assert got[2] == p[2] == ss and np.array_equal(got[0], p[0]) and np.array_equal(got[0], ms.cpu().numpy())
            np.testing.assert_allclose(got[1], p[1], atol=score_atol)
        assert sb == ss and np.array_equal(mb.cpu().numpy(), p[0])
    assert sum(len(p[0]) for p in plain) > 50


@pytest.mark.parametrize("profile", ["stop", "prune", "sharp"])
def test_encoded_sides_equal_plain_sides(b200_ctx, profile):
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, profile), ctx=b200_ctx)
    _check_encoded_equals_plain(fe)


def test_encoded_sides_on_simt_path():
    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "stop"), ctx=ctx)
        _check_encoded_equals_plain(fe)
    finally:
        ctx.close()


def test_encoded_sides_with_fp16_attention(b200_ctx):
    # one fp16 product per attention matmul: a different key split of the layer-0 self-attention moves scores by up to
    # ~5e-4 here (H100), within the ~1e-3 this mode agrees with the fp32-equivalent one; rows and stops stay identical
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), ctx=b200_ctx, fp16_attention=True)
    _check_encoded_equals_plain(fe, score_atol=1e-3)


def test_encoding_is_not_reused_across_modes(b200_ctx):
    """An image's encoding is made per front end (weights, kernel path) and attention numerics: switching either encodes
    again, and the results are those of the switched mode's per-pair matcher."""
    lg_sd = syn.lightglue_state_dict(2, "sharp")
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), lg_sd, ctx=b200_ctx)
    ims, pairs = _images()
    pairs = pairs[:4]
    fe.match_batch(pairs)
    fe.fp16_attention = 1
    got16 = fe.match_batch(pairs)
    assert len(ims[0].enc) == 2
    for (a, b), (m, s) in zip(pairs, got16):
        ms, ss = fe.match(a, b)
        assert s == ss and torch.equal(m, ms)
    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        simt = DeviceFrontEnd(syn.superpoint_state_dict(0), lg_sd, ctx=ctx)
        got = simt.match_batch(pairs)
        assert len(ims[0].enc) == 3
        for (a, b), (m, s) in zip(pairs, got):
            ms, ss = simt.match(a, b)
            assert s == ss and torch.equal(m, ms)
    finally:
        ctx.close()


def test_repeated_match_many_encodes_each_image_once(b200_ctx):
    """A second match_many over images that already have encodings launches no encoding work and returns the same rows."""
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), max_keypoints=500, ctx=b200_ctx)
    frames, _ = syn.synthetic_sequence(6, 240, 320)
    feats = fe.detect_many([torch.from_numpy(f).cuda() for f in frames])
    pairs = [(feats[i], feats[j]) for i in range(6) for j in range(i + 1, 6)]  # 15 pairs = 2 lock-step batches
    first = fe.match_many(pairs)
    assert all(len(f.enc) == 1 for f in feats)
    n0 = fe.launch_count()
    fe.profile_start("k_lg_posenc")  # runs only where an image enters the network from its features
    second = fe.match_many(pairs)
    _, n_posenc, _ = fe.profile_stop()
    n1 = fe.launch_count()
    third = fe.match_many(pairs)
    assert n_posenc == 0 and fe.launch_count() - n1 == n1 - n0
    for got in (second, third):
        for (m, s), (m0, s0) in zip(got, first):
            assert s == s0 and torch.equal(m, m0)
    assert sum(int(m.shape[0]) for m, _ in first) > 150
