"""GPU: with the attention output projection folded into the first feed-forward linear (weights.fold_message_projection),
LightGlue runs 3 k_gemm_ws launches per block (QKV or [to_qk; to_v], ffn.0, ffn.3) and SuperGlue 5 per GNN layer (q, k, v,
mlp.0, mlp.3): no launch forms the message any more.  The library refuses a blob whose projection slot was not folded."""
import ctypes as C

import numpy as np
import pytest
import torch

from gtsfm_b200 import _lib
from gtsfm_b200 import synthetic as syn
from gtsfm_b200 import weights
from gtsfm_b200.matcher import SuperGlueEngine
from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd

pytestmark = pytest.mark.gpu


def _feats(kp, d):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return DeviceFeatures(t(kp), t(np.ones(len(kp), np.float32)), t(d), (480, 640))


def _match_batched(fe, pairs):
    """One b2_lightglue_match_batched_dev call from the features (no encodings) -> its launch count."""
    arr = (_lib.LightGluePair * len(pairs))()
    outs = []
    for i, (a, b) in enumerate(pairs):
        m = torch.empty((min(len(a), len(b)), 2), dtype=torch.int64, device="cuda")
        s = torch.empty(len(m), dtype=torch.float32, device="cuda")
        outs.append((m, s))
        arr[i].kp0, arr[i].desc0, arr[i].n0 = a.kp.data_ptr(), a.desc.data_ptr(), len(a)
        arr[i].kp1, arr[i].desc1, arr[i].n1 = b.kp.data_ptr(), b.desc.data_ptr(), len(b)
        arr[i].enc0 = arr[i].enc1 = None
        arr[i].out_matches, arr[i].out_scores = m.data_ptr(), s.data_ptr()
    prm = _lib.LightGlueParams(0.95, 0.99, 0.1, fe.prune_min, fe.fp16_attention)
    n0 = fe.launch_count()
    fe.ctx.check(fe.lib.b2_lightglue_match_batched_dev(fe.ctx.handle, arr, len(pairs), C.byref(prm), fe._stream()), "match_batched_dev")
    torch.cuda.synchronize()
    return fe.launch_count() - n0


def _launches(fe, run, prefix):
    fe.profile_start(prefix)
    total = run()
    _, n, _ = fe.profile_stop()
    return int(n), total


def test_lightglue_lockstep_batch_runs_three_gemms_per_block(b200_ctx):
    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "bench"), max_keypoints=5000, ctx=b200_ctx)
    pairs = []
    for seed in range(8):
        kp0, _, d0, kp1, _, d1, _ = syn.synthetic_features(40 + seed, 700 + 50 * seed, 650 + 40 * seed)
        pairs.append((_feats(kp0, d0), _feats(kp1, d1)))
    run = lambda: _match_batched(fe, pairs)
    n = {p: _launches(fe, run, p) for p in ("k_gemm_ws", "k_gemm_ws/lg_self_", "k_gemm_ws/lg_self_qkv", "k_gemm_ws/lg_cross_",
                                             "k_gemm_ws/lg_cross_qv", "k_gemm_ws/lg_self_out", "k_gemm_ws/lg_cross_out", "k_gemm_ws/lg_assign_")}
    totals = {t for _, t in n.values()}
    assert len(totals) == 1, n  # every profiled run issued the same launches
    layers = n["k_gemm_ws/lg_self_qkv"][0]
    assert layers >= 1 and n["k_gemm_ws/lg_cross_qv"][0] == layers, n  # one lock-step launch per block and layer
    assert n["k_gemm_ws/lg_self_out"][0] == 0 and n["k_gemm_ws/lg_cross_out"][0] == 0, n
    assert n["k_gemm_ws/lg_self_"][0] == 3 * layers and n["k_gemm_ws/lg_cross_"][0] == 3 * layers, n
    assert n["k_gemm_ws"][0] == 6 * layers + n["k_gemm_ws/lg_assign_"][0], n


def test_superglue_runs_five_gemms_per_gnn_layer(b200_ctx):
    eng = SuperGlueEngine(syn.superglue_state_dict(1), ctx=b200_ctx)
    kp0, sc0, d0, kp1, sc1, d1, _ = syn.synthetic_features(5, 600, 700)
    run = lambda: eng.match(kp0, sc0, d0, kp1, sc1, d1, (480, 640, 3), (480, 640, 3))
    b200_ctx.profile_start("k_gemm_ws")
    run()
    _, n, _ = b200_ctx.profile_stop()
    assert n == 5 * weights.SUPERGLUE_GNN_LAYERS + 2  # + final_proj and the score matrix


def test_unfolded_blob_is_refused():
    ctx = _lib.Context(0)
    try:
        lg = weights._pack(syn.lightglue_state_dict(2), weights.LIGHTGLUE_ORDER)
        assert ctx.lib.b2_lightglue_set_weights(ctx.handle, _lib.ptr(lg), lg.size) == -2
        sg = weights._pack(weights.superglue_head_major(weights.fold_superglue_batchnorm(syn.superglue_state_dict(1))), weights.SUPERGLUE_ORDER)
        assert ctx.lib.b2_superglue_set_weights(ctx.handle, _lib.ptr(sg), sg.size) == -2
    finally:
        ctx.close()
