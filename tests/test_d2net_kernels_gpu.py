"""GPU: the pieces of the D2-Net path on their own, through the test-only entry points, plus the device-to-device handoff to
the two-way matcher.  Its convolutions (k_conv_ps<1> and the dilated k_conv_ps<2>) are tested with the other networks' in
tests/test_conv_ps_gpu.py.

* the AvgPool2d(2, stride=1) kernel against torch's avg_pool2d;
* the keypoint order (score descending, ties by (channel, row, column)) on candidates with many exactly equal scores;
* extract_many's device descriptors fed to TwoWayEngine.match_batched_dev against the host matcher, and the golden descriptors
  against the cv2 two-way reference under the float path's near-tie rule."""
import numpy as np
import pytest

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def test_avgpool_against_torch(b200_ctx):
    import torch
    import torch.nn.functional as F

    rng = np.random.default_rng(11)
    for H, W in ((9, 7), (2, 2), (31, 44)):
        x = np.maximum(rng.standard_normal((H, W, 256)), 0).astype(np.float32) * np.float32(3.0)
        out = np.empty((H - 1, W - 1, 256), np.float32)
        b200_ctx.check(b200_ctx.lib.b2_debug_d2net_avgpool_host(b200_ctx.handle, _lib.ptr(x), H, W, _lib.ptr(out)), "avgpool")
        want = F.avg_pool2d(torch.from_numpy(x).permute(2, 0, 1)[None], 2, stride=1)[0].permute(1, 2, 0).numpy()
        # the kernel sums in torch's order, so its fp32 result is torch's bit for bit; it hands that value to the next layer as
        # fp16 hi + lo planes (lo = fp16((v - hi) * 2^11)), which is what the entry point reads back.  Below fp16's normal
        # range (6.1e-5) hi is subnormal and the pair keeps ~1e-11 absolute, so the planes of torch's value are compared exactly.
        hi = want.astype(np.float16).astype(np.float32)
        lo = ((want - hi) * np.float32(2048.0)).astype(np.float16).astype(np.float32)
        assert np.array_equal(out, hi + lo * np.float32(1.0 / 2048.0)), np.abs(out - want).max()


def test_rank_orders_ties_by_channel_row_column(b200_ctx):
    rng = np.random.default_rng(3)
    n = 3000
    cells = rng.choice(512 * 400 * 400, n, replace=False)
    cij = np.stack([cells // 160000, cells // 400 % 400, cells % 400], 1).astype(np.int32)
    levels = np.array([0.5, 1.25, 1.2500001, 3.0, 7.75], np.float32)  # many exact ties, two scores one ulp apart
    scores = levels[rng.integers(0, len(levels), n)]
    scores[:50] = rng.random(50).astype(np.float32) + np.float32(10)
    want = np.lexsort((cij[:, 2], cij[:, 1], cij[:, 0], -scores.astype(np.float64)))
    for k in (n, 777, 1):
        order = np.full(min(n, k), -1, np.int32)
        rc = b200_ctx.lib.b2_debug_d2net_rank_host(b200_ctx.handle, _lib.ptr(scores), _lib.ptr(np.ascontiguousarray(cij)), n, k,
                                                   _lib.ptr(order))
        b200_ctx.check(rc, "rank")
        assert np.array_equal(order, want[:k])


def test_device_descriptors_feed_the_two_way_matcher(b200_ctx):
    import torch

    from gtsfm_b200.detector_descriptor import D2NetEngine
    from gtsfm_b200.matcher import TwoWayEngine

    eng = D2NetEngine(syn.d2net_state_dict(7), ctx=b200_ctx)
    tw = TwoWayEngine(ctx=b200_ctx)
    frames, _ = syn.synthetic_sequence(2, 240, 320)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    (x0, s0, d0, _), (x1, s1, d1, _) = eng.extract_many(dev, max_keypoints=2000)
    assert len(d0) > 50 and len(d1) > 50
    for ratio in (None, 0.8):
        m_dev = tw.match_batched_dev([(d0, d1)], ratio=ratio)[0].cpu().numpy()
        m_host = tw.match(d0.cpu().numpy(), d1.cpu().numpy(), ratio)
        assert np.array_equal(m_dev, m_host)
        assert len(m_dev) > 20
    # the two frames overlap: matched keypoints sit at about the same offset
    xy0, xy1 = x0.cpu().numpy()[m_dev[:, 0]], x1.cpu().numpy()[m_dev[:, 1]]
    shift = np.median(xy1 - xy0, axis=0)
    assert np.mean(np.linalg.norm(xy1 - xy0 - shift, axis=1) < 3.0) > 0.3


@pytest.mark.parametrize("ratio", [None, 0.8])
def test_golden_descriptors_against_twoway_reference(b200_ctx, golden_dir, ratio):
    from gtsfm_b200.matcher import TwoWayEngine
    from test_twoway_gpu import check_float_path

    a = np.load(golden_dir / "d2net_lund_1.npz")["desc"]
    b = np.load(golden_dir / "d2net_lund_2.npz")["desc"]
    check_float_path(TwoWayEngine(ctx=b200_ctx), a, b, ratio)
