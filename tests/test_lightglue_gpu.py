"""GPU parity: CUDA LightGlue (through the C ABI / plugin) vs golden fixtures from the reference and the CPU oracle.
Bar (BASELINE.json north_star): match indices exact."""
import pickle

import numpy as np
import pytest

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.gtsfm_api import Keypoints
from gtsfm_b200.matcher import B200LightGlueMatcher, LightGlueEngine

pytestmark = pytest.mark.gpu

_engines = {}


def engine(ctx, profile):
    if profile not in _engines:
        _engines[profile] = True
    return LightGlueEngine(syn.lightglue_state_dict(2, profile), ctx=ctx)


# bench_11 IS the configuration bench.py times: 5000 x 5000 keypoints, 'bench' weights, 9 full layers (79 key tiles x 160
# attention items through the stream-K split / fix-up); bench_12 the same weights at 1024 keypoints; full_15 has 6400
# columns in its final layer, more than the persistent assignment kernel holds (the multi-launch path)
@pytest.mark.parametrize("tag", ["full_5", "full_6", "prune_7", "stop_8", "prune_9", "stop_10", "bench_12", "bench_11", "full_15"])
def test_matches_equal_reference_fixture(b200_ctx, golden_dir, tag):
    fx = np.load(golden_dir / f"lightglue_{tag}.npz")
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(int(fx["seed"]), int(fx["n0"]), int(fx["n1"]))
    eng = engine(b200_ctx, str(fx["profile"]))
    m, sc = eng.match(kp0, d0, kp1, d1, return_scores=True)
    assert eng.last_stop == int(fx["stop"]), f"stop layer {eng.last_stop} vs reference {int(fx['stop'])}"
    assert m.dtype == np.int64 and m.shape == fx["matches"].shape, f"{m.shape} vs {fx['matches'].shape}"
    assert np.array_equal(m, fx["matches"])
    np.testing.assert_allclose(sc, fx["mscores"], atol=2e-4)


def test_bench_sequence_chain(b200_ctx, golden_dir):
    """The bench's own detect -> top-k -> match chain (frames 0 and 5 of its synthetic sequence, 'bench' weights, full depth):
    keypoints exact, then the reference-selected keypoints through describe + match give the reference's match rows."""
    from gtsfm_b200.detector_descriptor import SuperPointEngine

    fx = np.load(golden_dir / "pipeline_bench_seq_0_5.npz")
    frames, _ = syn.synthetic_sequence(8, 480, 640)
    sp = SuperPointEngine(syn.superpoint_state_dict(0), ctx=b200_ctx)
    lg = engine(b200_ctx, "bench")
    feats = []
    for f, key in ((frames[0], "a"), (frames[5], "b")):
        xy, sc = sp.detect(f)
        ref = fx[f"kp_{key}"].astype(np.float32)
        assert set(map(tuple, ref.tolist())) <= set(map(tuple, xy.tolist())), "reference-selected keypoints were not all detected"
        feats.append((ref, sp.describe(ref)))
    m = lg.match(feats[0][0], feats[0][1], feats[1][0], feats[1][1])
    assert lg.last_stop == int(fx["stop"]) == 9
    assert len(fx["matches"]) > 1000 and np.array_equal(m, fx["matches"].astype(np.int64))


@pytest.mark.parametrize("tag", ["full_5", "prune_7", "stop_8"])
def test_exact_fp32_simt_path(golden_dir, tag):
    """The exact-fp32 SIMT kernels (set_option force_simt: no tensor cores, no planes) are the on-device cross-check of the
    split-fp16 wgmma path; they must reproduce the same fixtures."""
    from gtsfm_b200 import _lib

    ctx = _lib.Context(0)
    try:
        ctx.set_option("force_simt", 1)
        fx = np.load(golden_dir / f"lightglue_{tag}.npz")
        kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(int(fx["seed"]), int(fx["n0"]), int(fx["n1"]))
        eng = LightGlueEngine(syn.lightglue_state_dict(2, str(fx["profile"])), ctx=ctx)
        m = eng.match(kp0, d0, kp1, d1)
        assert eng.last_stop == int(fx["stop"]) and np.array_equal(m, fx["matches"])
    finally:
        ctx.close()


def test_final_descriptors_match_oracle(b200_ctx):
    from oracle.lightglue_ref import lightglue_match

    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(21, 200, 180)
    sd = syn.lightglue_state_dict(2, "prune")
    tr = {}
    ref = lightglue_match(kp0, d0, kp1, d1, sd, trace=tr)
    eng = LightGlueEngine(sd, ctx=b200_ctx)
    m = eng.match(kp0, d0, kp1, d1)
    assert np.array_equal(m, ref)
    last = tr["stop"] - 1
    g0 = b200_ctx.debug_fetch("lg_desc0", 200 * 256).reshape(-1, 256)
    assert g0.shape == tr[f"desc0_l{last}"].shape
    np.testing.assert_allclose(g0, tr[f"desc0_l{last}"], atol=5e-5)


def test_lund_pair_and_crop_chain(b200_ctx, golden_dir):
    """detect -> wrapper top-k -> match on the lund-door frames vs the reference chain.

    The wrapper's top-k is `np.argpartition(-responses, k)` (gtsfm/common/keypoints.py:101-110): which keypoint sits at
    the k-th place, and hence every later index, flips on a 1-ulp score difference.  So the chain is compared (a) on
    the selected keypoint SET, allowing only swaps between scores within 1e-6 of the k-th score, and (b) on matches as
    coordinate pairs, which must be identical; where the selection is identical (the crop pair) raw indices must be too.
    """
    from gtsfm_b200.detector_descriptor import SuperPointEngine

    sp = SuperPointEngine(syn.superpoint_state_dict(0), ctx=b200_ctx)
    lg = LightGlueEngine(syn.lightglue_state_dict(2, "sharp"), ctx=b200_ctx)

    def feats(gray, k=5000):
        xy, sc = sp.detect(gray)
        sel = np.argpartition(-sc, k)[:k] if len(xy) > k else np.arange(len(xy))
        return xy[sel], sc[sel], sp.describe(xy[sel])

    def ref_feats(name):
        fx = np.load(golden_dir / f"superpoint_{name}.npz")
        sel = fx["topk_sel"]
        return fx["gray"], fx["keypoints"].astype(np.float32)[sel], fx["scores"][sel]

    g1, rkp1, rsc1 = ref_feats("lund1")
    g2, rkp2, rsc2 = ref_feats("lund2")
    fa, fb = feats(g1), feats(g2)
    for (kp, sc), (rkp, rsc) in (((fa[0], fa[1]), (rkp1, rsc1)), ((fb[0], fb[1]), (rkp2, rsc2))):
        mine, ref = set(map(tuple, kp.tolist())), set(map(tuple, rkp.tolist()))
        kth = np.sort(rsc)[0]
        swapped = [s for k_, s in zip(kp.tolist(), sc.tolist()) if tuple(k_) not in ref]
        assert len(mine ^ ref) <= 4 and all(abs(s - kth) < 1e-6 for s in swapped), (len(mine ^ ref), swapped, kth)
    fx = np.load(golden_dir / "lightglue_lund_1_2.npz")
    m = lg.match(fa[0], fa[2], fb[0], fb[2])
    assert lg.last_stop == int(fx["stop"])
    pairs = set(map(tuple, np.hstack([fa[0][m[:, 0]], fb[0][m[:, 1]]]).tolist()))
    ref_pairs = set(map(tuple, np.hstack([rkp1[fx["matches"][:, 0]], rkp2[fx["matches"][:, 1]]]).tolist()))
    assert len(fx["matches"]) > 100 and pairs == ref_pairs
    fxc = np.load(golden_dir / "pipeline_lund_crops_sharp.npz")
    ca, cb = np.ascontiguousarray(g1[0:1000, 0:700]), np.ascontiguousarray(g1[40:1040, 24:724])
    fa, fb = feats(ca), feats(cb)
    rka, rkb = fxc["kp_a"].astype(np.float32), fxc["kp_b"].astype(np.float32)
    for kp, rkp in ((fa[0], rka), (fb[0], rkb)):
        assert len(set(map(tuple, kp.tolist())) ^ set(map(tuple, rkp.tolist()))) <= 4
    m = lg.match(fa[0], fa[2], fb[0], fb[2])
    pairs = set(map(tuple, np.hstack([fa[0][m[:, 0]], fb[0][m[:, 1]]]).tolist()))
    ref_pairs = set(map(tuple, np.hstack([rka[fxc["matches"][:, 0]], rkb[fxc["matches"][:, 1]]]).tolist()))
    assert len(fxc["matches"]) > 500 and len(pairs ^ ref_pairs) <= 0.005 * len(ref_pairs), (len(pairs), len(ref_pairs), len(pairs ^ ref_pairs))


def test_plugin_contract(tmp_path, golden_dir):
    """tests/frontend/matcher/test_matcher_base.py:35-107 restated for the LightGlue plugin."""
    wpath = tmp_path / "superpoint_lightglue_v0-1_arxiv.pth"
    syn.save_pth(syn.lightglue_state_dict(2, "full"), wpath)
    matcher = B200LightGlueMatcher("superpoint", weights_path=wpath)
    pickle.dumps(matcher)
    kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(5, 300, 350)
    k0, k1 = Keypoints(kp0, responses=sc0), Keypoints(kp1, responses=sc1)
    m = matcher.match(k0, k1, d0, d1, (480, 640, 3), (480, 640, 3))
    pickle.dumps(matcher)
    assert m.dtype == np.int64 and m.ndim == 2 and m.shape[1] == 2
    assert np.array_equal(m, np.load(golden_dir / "lightglue_full_5.npz")["matches"])
    assert np.all(m[:, 0] < 300) and np.all(m[:, 1] < 350) and np.all(m >= 0)
    assert len(np.unique(m[:, 0])) == len(m) and len(np.unique(m[:, 1])) == len(m)  # one-to-one
    empty = Keypoints(np.zeros((0, 2), np.float32), responses=np.zeros(0, np.float32))
    assert matcher.match(empty, k1, np.zeros((0, 256), np.float32), d1, (480, 640, 3), (480, 640, 3)).size == 0
    assert matcher.match(k0, empty, d0, np.zeros((0, 256), np.float32), (480, 640, 3), (480, 640, 3)).size == 0
    with pytest.raises(ValueError):
        matcher.match(Keypoints(kp0), k1, d0, d1, (480, 640, 3), (480, 640, 3))


def test_feature_cache_is_opt_in_and_hashes_everything(b200_ctx, golden_dir):
    """b2_lightglue_match_host can keep device copies of host feature arrays (opt-in).  Off (default): every call uploads.
    On: a repeated call sends nothing, and ANY in-place edit - here ONE float in the middle of a descriptor array - is
    detected by the full-content hash and re-uploaded (a stale copy would silently change the matches)."""
    fx = np.load(golden_dir / "lightglue_full_5.npz")
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(int(fx["seed"]), int(fx["n0"]), int(fx["n1"]))
    eng = engine(b200_ctx, str(fx["profile"]))
    per_call = kp0.nbytes + d0.nbytes + kp1.nbytes + d1.nbytes
    sent = eng.h2d_bytes
    m0 = eng.match(kp0, d0, kp1, d1)
    m0b = eng.match(kp0, d0, kp1, d1)
    assert eng.h2d_bytes == sent + 2 * per_call, "cache off (default): both calls upload everything"
    assert np.array_equal(m0, fx["matches"]) and np.array_equal(m0b, m0)
    b200_ctx.set_option("feature_cache", 1)
    try:
        m1 = eng.match(kp0, d0, kp1, d1)
        sent = eng.h2d_bytes
        m2 = eng.match(kp0, d0, kp1, d1)
        assert np.array_equal(m1, fx["matches"]) and np.array_equal(m2, m1)
        assert eng.h2d_bytes == sent, "second call with the same arrays must not upload anything"
        # one float in the middle of the array, at a position no sampled signature would visit
        r, c = d1.shape[0] // 2 + 1, 131
        keep = d1[r].copy()
        d1[r, c] += 0.25
        eng.match(kp0, d0, kp1, d1)
        assert eng.h2d_bytes == sent + d1.nbytes, "an array edited in place must be sent again (and only that one)"
        # a visible edit: replace one matched descriptor row by its negative -> that match must disappear
        row = int(fx["matches"][len(fx["matches"]) // 2, 1])
        d1[r] = keep
        keep_row = d1[row].copy()
        d1[row] = -d1[row]
        m3 = eng.match(kp0, d0, kp1, d1)
        assert row not in set(m3[:, 1].tolist()) and row in set(m1[:, 1].tolist())
        d1[row] = keep_row
        m4 = eng.match(kp0, d0, kp1, d1)
        assert np.array_equal(m4, m1)
    finally:
        b200_ctx.set_option("feature_cache", 0)


@pytest.mark.parametrize("tag", ["full_5", "full_6", "stop_10"])
def test_fp16_attention_mode_vs_fp16_emulating_oracle(b200_ctx, golden_dir, tag):
    """Opt-in `fp16_attention` = the reference's CUDA numerics (lightglue.py:116-121: half q / k / v, fp16 flash SDPA, half
    result): ONE tensor-core product per attention matmul.  Pinned against an oracle that rounds the same operands and the
    result to fp16 (flash's internal rounding of the un-normalised probabilities cannot be emulated exactly): final
    descriptors within 4e-3, match sets nearly identical to both the emulating oracle and the fp32 fixture."""
    from oracle.lightglue_ref import lightglue_match

    fx = np.load(golden_dir / f"lightglue_{tag}.npz")
    kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(int(fx["seed"]), int(fx["n0"]), int(fx["n1"]))
    sd = syn.lightglue_state_dict(2, str(fx["profile"]))
    tr = {}
    ref16 = lightglue_match(kp0, d0, kp1, d1, sd, trace=tr, fp16_attention=True)
    eng = LightGlueEngine(sd, ctx=b200_ctx)
    m = eng.match(kp0, d0, kp1, d1, fp16_attention=True)

    def jaccard(a, b):
        sa, sb = set(map(tuple, a.tolist())), set(map(tuple, b.tolist()))
        return len(sa & sb) / max(1, len(sa | sb))

    assert jaccard(m, ref16) > 0.99, jaccard(m, ref16)
    assert jaccard(m, fx["matches"]) > 0.97, jaccard(m, fx["matches"])
    if eng.last_stop == tr["stop"] and tr["sizes"][-1][0] == int(fx["n0"]):  # nothing pruned: rows comparable one to one
        g0 = b200_ctx.debug_fetch("lg_desc0", int(fx["n0"]) * 256).reshape(-1, 256)
        ref = tr[f"desc0_l{tr['stop'] - 1}"]
        assert g0.shape == ref.shape and np.abs(g0 - ref).max() < 4e-3, np.abs(g0 - ref).max()
