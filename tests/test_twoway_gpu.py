"""GPU suite of the two-way matcher (csrc/mnn.cu): the exact path bit for bit against cv2, constructed ties, edge cases, the
float path's near-tie bound and the batched device entry point against per-pair host calls."""
import math

import numpy as np
import pytest

from oracle import twoway_ref

pytestmark = pytest.mark.gpu

EXACT = ["lund_stored", "sift", "orb"]
RATIOS = [("ratio", 0.8), ("noratio", None)]


@pytest.fixture(scope="module")
def engine(b200_ctx):
    from gtsfm_b200.matcher import TwoWayEngine

    return TwoWayEngine(ctx=b200_ctx)


def plugin(engine, ratio):
    from gtsfm_b200.matcher import B200TwoWayMatcher

    m = B200TwoWayMatcher(ratio_test_threshold=ratio)
    m._engine = engine
    return m


def run(engine, a, b, ratio):
    return plugin(engine, ratio).match(None, None, a, b, None, None)


def load(golden_dir, name):
    fx = np.load(golden_dir / f"twoway_{name}.npz")
    dt = str(fx["dtype"])
    return fx, fx["desc0"].astype(dt), fx["desc1"].astype(dt)


def assert_same_as_cv2(engine, a, b, ratio):
    ref, dref = twoway_ref.twoway_match(a, b, ratio)
    got = run(engine, a, b, ratio)
    assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref)
    if len(ref):
        _, d = engine.match(a, b, ratio, return_dist=True)
        assert np.array_equal(d.view(np.uint32), dref.view(np.uint32))


@pytest.mark.parametrize("name", EXACT)
@pytest.mark.parametrize("tag,ratio", RATIOS)
def test_exact_path_bit_identical_to_golden(engine, golden_dir, name, tag, ratio):
    fx, a, b = load(golden_dir, name)
    got = run(engine, a, b, ratio)
    assert got.dtype == np.uint32 and np.array_equal(got, fx[f"matches_{tag}"])
    m, d = engine.match(a, b, ratio, return_dist=True)
    assert np.array_equal(m, fx[f"matches_{tag}"].astype(np.int64))
    assert np.array_equal(d.view(np.uint32), fx[f"dist_{tag}"].view(np.uint32))


def squares(x, dim):
    """dim values in [0, 255] whose squares sum to x (greedy; the remainder shrinks fast)."""
    v = []
    while x > 0:
        t = min(255, math.isqrt(x))
        v.append(t)
        x -= t * t
    assert len(v) <= dim
    return np.array(v + [0] * (dim - len(v)), np.float32)


def test_ties_duplicates_all255_and_shared_sqrtf(engine):
    rng = np.random.default_rng(3)
    dim = 128
    # duplicate train rows: the lower index must win
    a = rng.integers(0, 256, (300, dim)).astype(np.float32)
    b = np.concatenate([a[::-1][:150], a[:200], a[:200]], 0)
    for ratio in (None, 0.8):
        assert_same_as_cv2(engine, a, b, ratio)
    # all-255 vectors on both sides
    a = np.full((40, dim), 255, np.float32)
    a[20:] = rng.integers(0, 256, (20, dim))
    b = np.concatenate([np.full((30, dim), 255, np.float32), a[25:]], 0)
    for ratio in (None, 0.8):
        assert_same_as_cv2(engine, a, b, ratio)
    # integer d^2 near 2^23 with one sqrtf: a zero query and a far one against train rows whose sums of squares are x + 1
    # and x, the larger at the lower index (below 124 * 255^2 so that the greedy split into squares fits in 128 values)
    xs = [x for x in range(7_950_000, 8_000_000) if np.sqrt(np.float32(x)) == np.sqrt(np.float32(x + 1))][:20]
    assert len(xs) == 20
    q = np.zeros((2, dim), np.float32)
    q[1, 126:] = 255
    t = np.stack([r for x in xs for r in (squares(x + 1, dim), squares(x, dim))], 0)
    qi, ti = q.astype(np.int64), t.astype(np.int64)
    d2 = ((qi * qi).sum(1)[:, None] + (ti * ti).sum(1)[None] - 2 * qi @ ti.T).astype(np.float64)  # exact integers
    for ratio in (None, 1.0):
        for x, y, dd in ((q, t, d2), (t, q, d2.T)):
            ref, _ = twoway_ref.twoway_match(x, y, ratio)
            # the arrays discriminate: a selection keyed on the integer d^2 instead of the float distance picks the other row
            assert not np.array_equal(twoway_ref.twoway_from_distances(np.ascontiguousarray(dd), ratio)[0], ref)
            assert_same_as_cv2(engine, x, y, ratio)


def test_reference_dummy_case(engine, golden_dir):
    fx, a, b = load(golden_dir, "dummy")
    assert np.array_equal(run(engine, a, b, 0.8), [[9, 5], [2, 4], [3, 2], [0, 3]])


def test_empty_inputs_and_no_match(engine):
    e = np.zeros((0, 128), np.float32)
    a = np.ones((5, 128), np.float32)
    for x, y in ((e, a), (a, e), (e, e)):
        r = run(engine, x, y, 0.8)
        assert r.shape == (0,) and r.dtype == np.float64
    # the ratio test rejects everything: every row is at the same non-zero distance from every row of the other side
    r = run(engine, a, np.full((3, 128), 2, np.float32), 0.5)
    assert r.shape == (0,) and r.dtype == np.float64
    assert twoway_ref.twoway_match(a, np.full((3, 128), 2, np.float32), 0.5)[0].shape == (0,)


def test_nan_rows_removed_and_remapped(engine, golden_dir):
    _, a, b = load(golden_dir, "sift")
    a, b = a[:800].copy(), b[:900].copy()
    a[[3, 100, 799]] = np.nan
    b[[0, 5]] = np.nan
    for ratio in (None, 0.8):
        ref, _ = twoway_ref.twoway_match(a, b, ratio)
        assert np.array_equal(run(engine, a, b, ratio), ref)


def test_ratio_with_one_candidate_raises(engine):
    a = np.ones((1, 16), np.float32)
    b = np.arange(48, dtype=np.float32).reshape(3, 16)
    for x, y in ((a, b), (b, a)):
        with pytest.raises(ValueError):
            twoway_ref.twoway_match(x, y, 0.8)
        with pytest.raises(ValueError):
            run(engine, x, y, 0.8)


def test_single_query_without_ratio(engine, golden_dir):
    _, a, b = load(golden_dir, "sift")
    for x, y in ((a[7:8], b), (a, b[11:12])):
        assert_same_as_cv2(engine, x, y, None)


def test_large_20000(engine):
    rng = np.random.default_rng(11)
    base = rng.integers(0, 120, (20000, 128))
    a = base.astype(np.float32)
    b = np.clip(base[rng.permutation(20000)] + rng.integers(-3, 4, base.shape), 0, 255).astype(np.float32)
    m, d = engine.match(a, b, 0.8, return_dist=True)
    ref, dref = twoway_ref.twoway_match(a, b, 0.8)
    assert len(ref) > 10000 and np.array_equal(m, ref.astype(np.int64)) and np.array_equal(d, dref)


def near_tie_rows(a, b, got, ref, ratio, tol=2.0 ** -18):
    """Rows of the symmetric difference of two match sets, and whether each is decided by a comparison that lies within
    `tol` relative of flipping in float64 distances (best vs second, the ratio test, or the mutual check's partner)."""
    a, b = a.astype(np.float64), b.astype(np.float64)
    D = np.sqrt(np.maximum((a * a).sum(1)[:, None] + (b * b).sum(1)[None] - 2 * a @ b.T, 0))

    def close(row):
        s = np.sort(row)
        if len(s) < 2:
            return False
        if s[1] - s[0] <= tol * max(s[0], 1e-30):
            return True
        return ratio is not None and abs(s[0] - ratio * s[1]) <= tol * max(s[0], 1e-30)

    diff = set(map(tuple, got.tolist())) ^ set(map(tuple, ref.tolist()))
    return diff, all(close(D[i]) or close(D[:, j]) for i, j in diff)


def check_float_path(engine, a, b, ratio):
    ref, _ = twoway_ref.twoway_match(a, b, ratio)
    got = run(engine, a, b, ratio)
    diff, ok = near_tie_rows(a, b, got.reshape(-1, 2), ref.reshape(-1, 2), ratio)
    assert len(diff) <= 0.001 * max(len(ref), 1) * 2, (len(diff), len(ref))
    assert ok, sorted(diff)[:10]
    if len(got):
        _, d = engine.match(a, b, ratio, return_dist=True)
        assert np.all(np.diff(d) >= 0)


@pytest.mark.parametrize("tag,ratio", RATIOS)
def test_float_path_kaze(engine, golden_dir, tag, ratio):
    _, a, b = load(golden_dir, "kaze")
    check_float_path(engine, a, b, ratio)


@pytest.mark.parametrize("tag,ratio", RATIOS)
def test_float_path_unit_512(engine, tag, ratio):
    rng = np.random.default_rng(5)
    a = rng.standard_normal((1500, 512))
    b = np.concatenate([a[:900] + 0.3 * rng.standard_normal((900, 512)), rng.standard_normal((700, 512))])
    a = (a / np.linalg.norm(a, axis=1, keepdims=True)).astype(np.float32)
    b = (b / np.linalg.norm(b, axis=1, keepdims=True)).astype(np.float32)
    check_float_path(engine, a, b, ratio)


@pytest.mark.parametrize("ratio", [None, 0.8])
def test_batched_dev_equals_host_calls(engine, golden_dir, ratio):
    import torch

    rng = np.random.default_rng(9)
    _, s0, s1 = load(golden_dir, "sift")
    _, k0, k1 = load(golden_dir, "kaze")
    _, o0, o1 = load(golden_dir, "orb")
    _, d0, d1 = load(golden_dir, "dummy")
    f128 = (rng.random((600, 128)) * 40).astype(np.float32)  # not integer-valued: shares the (128, float32) call with SIFT
    u0 = rng.standard_normal((700, 512)).astype(np.float32)
    u1 = rng.standard_normal((900, 512)).astype(np.float32)
    pairs = [(s0, s1), (f128, s1[:800]), (k0[:1000], k1), (d0, d1), (u0, u1), (o0, o1), (s0[:0], s1[:50]), (s0[:1000], s1[500:3000]),
             (k0[:300], k1[:700]), (o0[:130], o1[:4000 // 2])]
    dev = [(torch.from_numpy(np.ascontiguousarray(x)).cuda(), torch.from_numpy(np.ascontiguousarray(y)).cuda()) for x, y in pairs]
    res = engine.match_batched_dev(dev, ratio, return_dist=True)
    torch.cuda.synchronize()
    for (x, y), (m, d) in zip(pairs, res):
        hm, hd = engine.match(x, y, ratio, return_dist=True)
        assert np.array_equal(m.cpu().numpy(), hm)
        assert np.array_equal(d.cpu().numpy().view(np.uint32), hd.view(np.uint32))
