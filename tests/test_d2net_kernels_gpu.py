"""GPU: the pieces of the D2-Net path on their own, through the test-only entry points, plus the device-to-device handoff to
the two-way matcher.

* k_conv_ps<2> (3x3, dilation 2, padding 2) and k_conv_ps<1> against torch's float64 conv2d on random NHWC planes, at shapes that
  are not multiples of the 16 x 8 tile;
* the AvgPool2d(2, stride=1) kernel against torch's avg_pool2d;
* the keypoint order (score descending, ties by (channel, row, column)) on candidates with many exactly equal scores;
* extract_many's device descriptors fed to TwoWayEngine.match_batched_dev against the host matcher, and the golden descriptors
  against the cv2 two-way reference under the float path's near-tie rule."""
import numpy as np
import pytest

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _conv(ctx, x, w, b, dil, relu):
    H, W, cin = x.shape
    cout = w.shape[0]
    out = np.empty((H, W, cout), np.float32)
    rc = ctx.lib.b2_debug_conv_ps_host(ctx.handle, dil, _lib.ptr(np.ascontiguousarray(x)), H, W, cin, cout, _lib.ptr(np.ascontiguousarray(w)),
                                       _lib.ptr(np.ascontiguousarray(b)), relu, _lib.ptr(out))
    ctx.check(rc, "debug_conv_ps_host")
    return out


@pytest.mark.parametrize("dil,H,W,cin,cout,relu", [(2, 37, 29, 256, 512, 1), (2, 13, 21, 512, 512, 1), (2, 5, 3, 64, 128, 0),
                                                   (2, 70, 45, 128, 64, 0), (1, 37, 29, 256, 128, 1)])
def test_conv_ps_against_conv2d(b200_ctx, dil, H, W, cin, cout, relu):
    import torch
    import torch.nn.functional as F

    rng = np.random.default_rng(H * 1000 + W + dil)
    x = np.maximum(rng.standard_normal((H, W, cin)), 0).astype(np.float32)  # post-ReLU activations, as in the network
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b = (0.05 * rng.standard_normal(cout)).astype(np.float32)
    got = _conv(b200_ctx, x, w, b, dil, relu)
    t = lambda a: torch.from_numpy(a).double()  # noqa: E731
    want = F.conv2d(t(x).permute(2, 0, 1)[None], t(w), t(b), padding=dil, dilation=dil)[0].permute(1, 2, 0)
    if relu:
        want = F.relu(want)
    want = want.numpy()
    # fp32 torch on the same operands: the rounding a plain float32 convolution has
    f32 = F.conv2d(torch.from_numpy(x).permute(2, 0, 1)[None], torch.from_numpy(w), torch.from_numpy(b), padding=dil, dilation=dil)[0]
    f32 = (F.relu(f32) if relu else f32).permute(1, 2, 0).numpy()
    scale = np.abs(want).max()
    err, err32 = np.abs(got - want).max() / scale, np.abs(f32 - want).max() / scale
    print(f"dil {dil} {H}x{W} {cin}->{cout}: max err {err:.2e} of max |y| (fp32 torch {err32:.2e})")
    assert err < 1e-5, err


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
