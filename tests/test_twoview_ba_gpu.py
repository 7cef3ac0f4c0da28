"""GPU: the device two-view refinement (csrc/twoview_ba.cu, b2_twoview_ba_batched_dev) against oracle/twoview_ba_ref.py -
triangulation, two-view bundle adjustment, the 0.5 px filter and inlier support - on the seeded scenes of
tests/golden/twoview_ba_scenes.npz and on lund-door's 66 pairs as the device verifier hands them over."""
import numpy as np
import pytest
import torch

from gtsfm_b200 import synthetic as syn
from gtsfm_b200.pipeline import DeviceFeatures, DeviceFrontEnd, RefineOptions
from gtsfm_b200.two_view import B200TwoViewBatch
from oracle import twoview_ba_ref as ref

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-6       # rad
TRACE_RTOL = 1e-9
BORDER_PX = 1e-6     # a track this close to the 0.5 px threshold may fall either way
MAX_BORDER = 2       # such tracks allowed over a whole test


def _border_rows(diff, track_rows, track_err):
    """The rows in which device and oracle differ must be tracks within BORDER_PX of the threshold -> their count."""
    err = dict(zip(track_rows.tolist(), track_err.tolist()))
    for r in diff:
        assert abs(err.get(int(r), np.inf) - 0.5) < BORDER_PX, f"row {r} differs and is not at the threshold"
    return len(diff)


def _angle(Ra, Rb):
    return float(np.arccos(np.clip((np.trace(Ra.T @ Rb) - 1.0) / 2.0, -1.0, 1.0)))


def _dir_angle(a, b):
    return float(np.arccos(np.clip(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)), -1.0, 1.0)))


@pytest.fixture(scope="module")
def fe():
    return DeviceFrontEnd(syn.superpoint_state_dict(0), max_keypoints=64)


@pytest.fixture(scope="module")
def scenes(golden_dir):
    z = np.load(golden_dir / "twoview_ba_scenes.npz")
    return {str(n): {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(f"{n}/")} for n in z["names"]}


def _item(s):
    """One scene as refine_many's input: keypoints = the scene's pixels, matches = identity rows, the verified mask."""
    k = int(s["k"])
    kp1 = torch.from_numpy(s["uv1"].astype(np.float32)).cuda()
    kp2 = torch.from_numpy(s["uv2"].astype(np.float32)).cuda()
    a = DeviceFeatures(kp1, torch.zeros(k, device="cuda"), torch.zeros((k, 1), device="cuda"), (480, 640))
    b = DeviceFeatures(kp2, torch.zeros(k, device="cuda"), torch.zeros((k, 1), device="cuda"), (480, 640))
    m = torch.arange(k, device="cuda", dtype=torch.int64)[:, None].repeat(1, 2).contiguous()
    mask = torch.zeros(k, dtype=torch.uint8, device="cuda")
    mask[torch.from_numpy(s["verified"]).cuda()] = 1
    item = (a, b, m, tuple(s["cal1"]), tuple(s["cal2"]))
    ver = (np.eye(3), s["R0"], s["t0"], len(s["verified"]), mask)
    return item, ver


def _run(fe, scene_list, trace=False):
    items, vers = zip(*[_item(s) for s in scene_list])
    out = fe.refine_many(list(items), list(vers), RefineOptions(), trace=trace)
    torch.cuda.synchronize()
    return out


def _check_against_oracle(name, s, R, t, rows, res, trace_row=None):
    ok = bool(s["out_ok"])
    assert (R is not None) == ok, f"{name}: success {R is not None}, oracle {ok}"
    if not ok:
        return 0
    assert _angle(R, s["out_R"]) < ROT_TOL, name
    assert _dir_angle(t, s["out_t"]) < ROT_TOL, name
    got = rows[:, 0].cpu().numpy() if rows is not None and len(rows) else np.zeros(0, np.int64)
    want = s["out_rows"]
    diff = np.setxor1d(got, want)
    if trace_row is not None and len(s["out_trace"]):
        assert res.trace_len == len(s["out_trace"]), f"{name}: {res.trace_len} LM records, oracle {len(s['out_trace'])}"
        np.testing.assert_allclose(trace_row[:res.trace_len], s["out_trace"], rtol=TRACE_RTOL, atol=1e-12, err_msg=name)
    return _border_rows(diff, s["out_track_rows"], s["out_track_err"])


def test_every_scene_equals_the_oracle(fe, scenes):
    """Success / failure, R and t to 1e-6 rad, the kept rows, and (for the pairs that succeed) the LM cost trace to 1e-9
    relative, scene by scene.  The pure-rotation scene fails both ways; its LM path is not compared: with no baseline the
    Hessian is near-singular and rounding differences change the trajectory."""
    border = 0
    for name, s in scenes.items():
        (out, tr) = _run(fe, [s], trace=True)
        R, t, rows, res = out[0]
        border += _check_against_oracle(name, s, R, t, rows, res, tr[0])
    assert border <= MAX_BORDER, f"{border} kept rows differ from the oracle"


def test_batches_equal_one_pair_at_a_time(fe, scenes):
    """Batches of 1, 8 and 33 pairs (the scenes repeated) give what each pair gives alone, bit for bit."""
    names = sorted(scenes)
    alone = {n: _run(fe, [scenes[n]]) [0] for n in names}
    for size in (1, 8, 33):
        batch = [names[i % len(names)] for i in range(size)]
        out = _run(fe, [scenes[n] for n in batch])
        for n, (R, t, rows, res) in zip(batch, out):
            R1, t1, rows1, res1 = alone[n]
            assert (R is None) == (R1 is None), n
            if R is None:
                continue
            assert np.array_equal(R, R1) and np.array_equal(t, t1), n
            assert torch.equal(rows, rows1), n
            assert res.iterations == res1.iterations and res.final_error == res1.final_error, n


def test_default_off_returns_the_verification(fe):
    """bundle_adjust_2view defaults to off: B200TwoViewBatch returns verify_many's rows, pose and ratio unchanged."""
    fe2 = DeviceFrontEnd(syn.superpoint_state_dict(0), syn.lightglue_state_dict(2, "sharp"), max_keypoints=1024)
    frames, cal = syn.synthetic_sequence(4, 240, 320)
    feats = {i: fe2.detect(torch.from_numpy(f).cuda()) for i, f in enumerate(frames)}
    pairs = [(0, 1), (0, 2), (1, 3), (2, 3)]
    intr = {i: cal for i in feats}
    batch = B200TwoViewBatch(fe2, 4.0)
    assert batch.refine is None
    res = batch.run(feats, pairs, intr)
    for (i1, i2) in pairs:
        m, _ = fe2.match(feats[i1], feats[i2])
        E, R, t, n, mask = fe2.verify_many([(feats[i1], feats[i2], m, cal, cal)])[0]
        r = res[(i1, i2)]
        if E is None:
            assert r.i2Ri1 is None
            continue
        assert np.array_equal(r.v_corr_idxs, m[mask.bool()].cpu().numpy())
        assert np.array_equal(r.i2Ri1.matrix(), R) and r.inlier_ratio_est_model == n / len(m)


def test_lund_door_66_pairs_equal_the_oracle(fe, golden_dir):
    """B200TwoViewBatch(bundle_adjust_2view=True) on lund-door's 66 pairs: the verifier still hands over the rows and pose
    tests/golden/twoview_ba_lund_door.npz stores, and the refinement of them equals the oracle's (success, R and t to 1e-6
    rad, the kept rows, the LM cost trace of the pairs that succeed)."""
    from oracle import make_golden_twoview_ba as mg

    kps, pairs, rows, cal = mg.lund_inputs()
    z = np.load(golden_dir / "twoview_ba_lund_door.npz")
    feats = {i: DeviceFeatures(torch.from_numpy(k).cuda(), torch.zeros(len(k), device="cuda"), torch.zeros((len(k), 1), device="cuda"),
                               (0, 0)) for i, k in kps.items()}
    put = {p: torch.from_numpy(m).cuda() for p, m in rows.items()}
    intr = {i: cal for i in kps}
    pre = B200TwoViewBatch(fe, 4.0).run(feats, pairs, intr, put)
    post = B200TwoViewBatch(fe, 4.0, bundle_adjust_2view=True).run(feats, pairs, intr, put)
    n_ok = border = 0
    items, vers, keys = [], [], []
    for p in pairs:
        key, m = f"{p[0]}_{p[1]}", rows[p]
        v, r = pre[p], post[p]
        assert (v.i2Ri1 is not None) == bool(z[f"{key}/ok"]), p
        if v.i2Ri1 is None:
            assert r.i2Ri1 is None, p
            continue
        row_of = {tuple(x): j for j, x in enumerate(m)}
        assert np.array_equal(sorted(row_of[tuple(x)] for x in v.v_corr_idxs), z[f"{key}/verified"]), p
        assert np.array_equal(v.i2Ri1.matrix(), z[f"{key}/R0"]), p
        assert (r.i2Ri1 is not None) == bool(z[f"{key}/out_ok"]), p
        assert r.inlier_ratio_est_model == v.inlier_ratio_est_model
        if r.i2Ri1 is None:
            continue
        n_ok += 1
        assert _angle(r.i2Ri1.matrix(), z[f"{key}/out_R"]) < ROT_TOL, p
        assert _dir_angle(r.i2Ui1.point3(), z[f"{key}/out_t"]) < ROT_TOL, p
        diff = np.setxor1d([row_of[tuple(x)] for x in r.v_corr_idxs], z[f"{key}/out_rows"])
        border += _border_rows(diff, z[f"{key}/out_track_rows"], z[f"{key}/out_track_err"])
        keys.append(key)
        item, ver = _item(dict(uv1=kps[p[0]][m[:, 0]], uv2=kps[p[1]][m[:, 1]], k=len(m), verified=z[f"{key}/verified"],
                               cal1=np.array(cal), cal2=np.array(cal), R0=z[f"{key}/R0"], t0=z[f"{key}/t0"]))
        items.append(item)
        vers.append(ver)
    assert n_ok >= 30, f"only {n_ok} of 66 pairs survived refinement"
    assert border <= MAX_BORDER, f"{border} kept rows differ from the oracle"
    out, tr = fe.refine_many(items, vers, RefineOptions(), trace=True)
    for key, (_, _, _, res), row in zip(keys, out, tr):
        want = z[f"{key}/out_trace"]
        assert res.trace_len == len(want), key
        np.testing.assert_allclose(row[:res.trace_len], want, rtol=TRACE_RTOL, atol=1e-12, err_msg=key)
