"""GPU: the D2-Net detector-descriptor (b2_d2net_*) against the goldens made by the unmodified reference plugin, plus the
properties of the device path.

Keypoints are paired with the golden's by position.  A keypoint present on one side only is accepted only when the golden's
margin for its cell (the relative distance of the cell's strongest channel to the nearest detection decision) is below
1e-5.  Positions and descriptors must be within 20x the fp32-vs-fp64 spread the generator recorded for the case.  Scores
get the larger of that and 1e-4 relative: the split-fp16 convolutions (conv_ps.cuh) are about fp32 per product but not
fp32-rounded per layer, and over nine layers they leave the scores ~2.4e-5 relative from fp32 on an H100, above 20x the
spread (~1e-5); DESIGN.md section 3 records the measured maxima.  The output order must be the golden's wherever two
neighbouring golden scores are further apart than that tolerance."""
import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from oracle import d2net_ref

pytestmark = pytest.mark.gpu
SEED = 7
FLOOR_SCORE_REL = 1e-4


@pytest.fixture(scope="module")
def engine(b200_ctx):
    from gtsfm_b200.detector_descriptor import D2NetEngine

    return D2NetEngine(syn.d2net_state_dict(SEED), ctx=b200_ctx)


def _cell(xy):  # feature-map cell of an output position: |step| < 0.5 around it
    fi = ((xy[:, 1] - 0.5) / 2 - 0.5) / 2
    fj = ((xy[:, 0] - 0.5) / 2 - 0.5) / 2
    return np.rint(fi).astype(int), np.rint(fj).astype(int)


@pytest.mark.parametrize("name", d2net_ref.CASES)
def test_golden(engine, golden_dir, name):
    from scipy.spatial import cKDTree

    z = np.load(golden_dir / f"d2net_{name}.npz")
    arr = d2net_ref.case_image(name, golden_dir)
    xy, sc, desc = engine.detect_and_describe(arr, int(z["max_keypoints"]))
    assert np.all(np.diff(sc.astype(np.float64)) <= 0)
    assert np.allclose(np.linalg.norm(desc, axis=1), 1, atol=1e-5)
    gxy, gsc, gdesc, margin = z["xy"], z["scores"], z["desc"], z["margin"]
    tol_xy, tol_d = 20 * float(z["spread_xy"]), 20 * float(z["spread_desc"])
    tol_sc = max(20 * float(z["spread_score_rel"]), FLOOR_SCORE_REL)
    dist, nn = cKDTree(xy).query(gxy, distance_upper_bound=tol_xy) if len(xy) else (np.full(len(gxy), np.inf), None)
    found = np.isfinite(dist)
    ci, cj = _cell(gxy[~found])
    assert np.all(margin[ci, cj] < 1e-5), f"{name}: {int((~found).sum())} golden keypoints missing"
    extra = np.setdiff1d(np.arange(len(xy)), nn[found]) if len(xy) else np.zeros(0, int)
    ci, cj = _cell(xy[extra])
    assert np.all(margin[ci, cj] < 1e-5), f"{name}: {len(extra)} keypoints not in the golden"
    g = np.flatnonzero(found)
    o = nn[found]
    if len(g):
        rel = np.abs(sc[o] - gsc[g]) / np.abs(gsc[g])
        print(f"{name}: {len(xy)}/{len(gxy)} keypoints, max |dxy| {dist[found].max():.2e} (tol {tol_xy:.1e}), "
              f"score rel {rel.max():.2e} (tol {tol_sc:.1e}, 20x spread {20 * float(z['spread_score_rel']):.1e})", end="")
        assert rel.max() <= tol_sc
        kd = g < len(gdesc)
        if kd.any():
            dd = np.abs(desc[o[kd]] - gdesc[g[kd]]).max()
            print(f", desc {dd:.2e} (tol {tol_d:.1e}, 20x spread {20 * float(z['spread_desc']):.1e})")
            assert dd <= tol_d
        # order: where the device puts golden keypoints out of the golden's order, their golden scores must be within tolerance
        g_by_device = g[np.argsort(o)]
        back = np.flatnonzero(np.diff(g_by_device) < 0)
        a, b = gsc[g_by_device[back]], gsc[g_by_device[back + 1]]
        assert np.all(np.abs(a - b) <= tol_sc * np.abs(a)), f"{name}: {len(back)} order inversions beyond the score tolerance"


def test_top_k_is_a_prefix(engine, golden_dir):
    arr = d2net_ref.case_image("lund_1", golden_dir)
    xy, sc, desc = engine.detect_and_describe(arr, 5000)
    for k in (0, 1, 100, 2000):
        xk, sk, dk = engine.detect_and_describe(arr, k)
        assert len(sk) == min(k, len(sc))
        assert np.array_equal(xk, xy[:k]) and np.array_equal(sk, sc[:k]) and np.array_equal(dk, desc[:k])
    # the order of exactly equal scores is checked on the rank kernel itself (test_d2net_kernels_gpu.py)


def test_layouts_batches_and_runs_agree(engine, golden_dir):
    import torch

    a = d2net_ref.case_image("lund_1", golden_dir)[:600, :700].copy()
    b = d2net_ref.case_image("lund_2", golden_dir)[:600, :700].copy()
    ref = [engine.detect_and_describe(x, 3000) for x in (a, b)]
    for x, r in zip((a[:, :, None], np.repeat(a[:, :, None], 3, axis=2)), (ref[0], ref[0])):
        got = engine.detect_and_describe(x, 3000)
        assert all(np.array_equal(p, q) for p, q in zip(got, r))
    again = engine.detect_and_describe(a, 3000)
    assert all(np.array_equal(p, q) for p, q in zip(again, ref[0]))
    dev = torch.device("cuda", 0)
    padded = torch.zeros((2, 600, 768), dtype=torch.uint8, device=dev)  # row pitch 768 > 700
    padded[0, :, :700] = torch.from_numpy(a).to(dev)
    padded[1, :, :700] = torch.from_numpy(b).to(dev)
    out = engine.extract_many([padded[0, :, :700], padded[1, :, :700]], max_keypoints=3000)
    torch.cuda.synchronize()
    for (xy, sc, de, total), r in zip(out, ref):
        assert total >= len(r[1])
        assert np.array_equal(xy.cpu().numpy(), r[0]) and np.array_equal(sc.cpu().numpy(), r[1]) and np.array_equal(de.cpu().numpy(), r[2])


def test_small_and_out_of_range_inputs(engine, b200_ctx):
    from gtsfm_b200 import _lib

    xy, sc, desc = engine.detect_and_describe(np.full((8, 8), 77, np.uint8), 10)
    assert xy.shape[1] == 2 and desc.shape[1] == 512 and len(sc) == len(xy)
    xy, sc, desc = engine.detect_and_describe(syn.synthetic_frame(5, 64, 64), 0)
    assert xy.shape == (0, 2) and desc.shape == (0, 512)
    img = np.zeros((1601, 16), np.uint8)
    xyb, scb, deb = np.empty((4, 2), np.float32), np.empty(4, np.float32), np.empty((4, 512), np.float32)
    n = _lib.C.c_int(0)
    for h, w in ((1601, 16), (1500, 1400), (7, 64)):
        rc = b200_ctx.lib.b2_d2net_detect_host(b200_ctx.handle, _lib.ptr(img), h, w, 1, 4, _lib.ptr(xyb), _lib.ptr(scb), _lib.ptr(deb),
                                                _lib.C.byref(n), None)
        assert rc == -2, (h, w, rc)


def test_force_simt_refuses():
    from gtsfm_b200 import _lib
    from gtsfm_b200.detector_descriptor import D2NetEngine

    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        with pytest.raises(_lib.B200Error, match=r"\(-3\)"):
            D2NetEngine(syn.d2net_state_dict(SEED), ctx=ctx)
    finally:
        ctx.close()


def test_plugin_drop_in(engine, golden_dir):
    from gtsfm_b200.detector_descriptor import B200D2NetDetectorDescriptor
    from gtsfm_b200.gtsfm_api import Image

    p = B200D2NetDetectorDescriptor(max_keypoints=300, model_path=syn.d2net_state_dict(SEED))
    p._engine = engine
    arr = d2net_ref.case_image("synthetic", golden_dir)
    kp, desc = p.detect_and_describe(Image(arr))
    xy, sc, de = engine.detect_and_describe(arr, 300)
    assert len(kp) == 300 and desc.shape == (300, 512) and desc.dtype == np.float32
    assert np.array_equal(kp.coordinates, xy) and np.array_equal(kp.responses, sc) and kp.scales is None
    assert np.array_equal(desc, de)
