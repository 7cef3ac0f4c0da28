"""GPU: DeviceFrontEnd's lanes (the extra library contexts behind detect_many, match_superglue_many and verification) are
configured like the front end's own context: options set on it before the lanes exist reach every lane."""
import ctypes

import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn
from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd
from gtsfm_b200.verifier import E_MAX_ITERS, ransac_problem
from oracle import verifier_ref as vr

pytestmark = pytest.mark.gpu


def _launches(fe, prefix, fn):
    fe.profile_start(prefix)
    out = fn()
    torch.cuda.synchronize()
    return out, fe.profile_stop()[1]


def test_detect_lanes_follow_force_simt(monkeypatch):
    """Every detect_many lane runs the exact-fp32 SIMT SuperPoint, as the front end's context does: the same bits as detect,
    and no tensor-core convolution anywhere."""
    from gtsfm_b200 import pipeline

    monkeypatch.setattr(pipeline, "DETECT_LANES", 4)
    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        fe = DeviceFrontEnd(syn.superpoint_state_dict(0), None, max_keypoints=400, ctx=ctx)
        frames, _ = syn.synthetic_sequence(5, 240, 320)
        imgs = [torch.from_numpy(f).cuda() for f in frames]
        fe.detect_many(imgs)  # makes the lanes
        assert len(fe._all_ctx()) == 4
        ref = [fe.detect(im) for im in imgs]
        got, n_tc = _launches(fe, "k_conv_ps", lambda: fe.detect_many(imgs))
        assert n_tc == 0
        for r, g in zip(ref, got):
            assert len(r) > 0 and torch.equal(g.kp, r.kp) and torch.equal(g.score, r.score) and torch.equal(g.desc, r.desc)
    finally:
        ctx.close()


def test_superglue_lanes_follow_force_simt(monkeypatch):
    from gtsfm_b200 import pipeline

    monkeypatch.setattr(pipeline, "SG_LANES", 3)
    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        fe = DeviceFrontEnd(syn.superpoint_state_dict(0), None, max_keypoints=300, ctx=ctx,
                            superglue_sd=syn.superglue_state_dict(1, "sharp"))
        frames, _ = syn.synthetic_sequence(4, 240, 320)
        feats = fe.detect_many([torch.from_numpy(f).cuda() for f in frames])
        pairs = [(feats[i], feats[j]) for i in range(4) for j in range(i + 1, 4)]
        fe.match_superglue_many(pairs)  # makes the lanes
        ref = [fe.match_superglue(a, b) for a, b in pairs]
        got, n_gemm = _launches(fe, "k_gemm_ws", lambda: fe.match_superglue_many(pairs))
        again, n_flash = _launches(fe, "k_flash_ps", lambda: fe.match_superglue_many(pairs))
        assert n_gemm == 0 and n_flash == 0
        for r, g, h in zip(ref, got, again):
            assert torch.equal(g, r) and torch.equal(h, r)
        assert sum(len(r) for r in ref) > 50 and len(fe._lanes["superglue"]) == 3
    finally:
        ctx.close()


def test_verify_lane_follows_ransac_workspace(b200_ctx):
    """ransac_workspace_mb on the front end's context cuts verify_many_async's batch into the sub-batches b2_ransac_plan gives
    for that budget (an E problem at 2000 points needs 3.4 MB, so 1 MiB runs each alone); the results are those of the
    default budget."""
    items = []
    for i, (k, ratio) in enumerate([(2000, 0.3), (2000, 0.6), (1500, 0.5), (4, 1.0), (2000, 0.45)]):
        kp1, kp2, _, K, *_ = vr.synthetic_two_view(800 + i, max(k, 1), ratio)
        f = [DeviceFeatures(torch.from_numpy(kp[:k].astype(np.float32)).cuda(), torch.zeros(k, device="cuda"),
                            torch.zeros(k, 256, device="cuda"), (960, 1280)) for kp in (kp1, kp2)]
        rows = torch.arange(k, device="cuda", dtype=torch.int64)[:, None].repeat(1, 2).contiguous()
        items.append((f[0], f[1], rows, K, K))
    masks = [torch.zeros(len(a), dtype=torch.uint8, device="cuda") for a, *_ in items]
    probs = [ransac_problem(len(a), 0, 4.0 / cal[0], E_MAX_ITERS, mask=mask, kp1=a.kp, kp2=b.kp, matches=m, cal1=cal, cal2=cal)
             for (a, b, m, cal, _), mask in zip(items, masks) if len(a) >= 6]  # the problems verify_many hands to the library
    first = (ctypes.c_int * (len(probs) + 1))()
    sub_batches = b200_ctx.lib.b2_ransac_plan((_lib.RansacProblem * len(probs))(*probs), len(probs), 1 << 20, first)
    assert sub_batches == len(probs) == 4

    sp_sd = syn.superpoint_state_dict(0)
    torch.cuda.synchronize()
    ref = DeviceFrontEnd(sp_sd, ctx=b200_ctx).verify_many_async(items).result()
    ctx = _lib.Context(0)
    try:
        ctx.set_option("ransac_workspace_mb", 1)
        fe = DeviceFrontEnd(sp_sd, ctx=ctx)
        fe.verify_many_async(items[:1]).result()  # makes the verification lane
        s0 = fe._vctx.ransac_sync_count()
        got = fe.verify_many_async(items).result()
        assert fe._vctx.ransac_sync_count() - s0 == sub_batches
        assert sum(r[0] is not None for r in ref) == 4
        for r, g in zip(ref, got):
            assert (r[0] is None) == (g[0] is None) and r[3] == g[3]
            if r[0] is not None:
                assert all(np.array_equal(x, y) for x, y in zip(r[:3], g[:3]))
            assert torch.equal(r[4], g[4])
    finally:
        ctx.close()
