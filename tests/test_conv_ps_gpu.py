"""GPU: the shared 3x3 convolution layer (k_conv_ps<1> / <2> through conv_ps_run, and the exact-fp32 SIMT k_conv3x3), through
b2_debug_conv_host, in every mode its callers use, against fp64 (oracle/conv_ref.py) and bit for bit against itself.

Each row of CASES stands for one kind of layer a network launches (its Cin -> Cout, pool, ReLU, dilation and outputs), at a
spatial size scaled down so the fp64 reference stays cheap, chosen to reach the edges: partial 16 x 8 tiles in both directions,
odd sizes under the pool, images smaller than one tile (1 x 1, 2 x 2, 3 x 5, 1 x N and N x 1; 16 x 16 is NetVLAD's smallest
input, which reaches conv4_3 at 2 x 2 and conv5_x at 1 x 1), and one size with far more tiles than CTAs.  Rows with Cin = 64
keep the CTA's weights resident across its tiles; Cin >= 128 reloads them per 64-channel chunk.

Tolerance (oracle/conv_ref.py derives it): with S = conv(|x|, |w|) over K = 9 Cin products, 16 * 2^-22 * S for the operand
split, (K / 16) * 2^-23 * S for the truncating accumulation, 2^-23 * S for joining the accumulators, the largest of the four
under a pool, plus 2^-23 |y| for the bias add; the SIMT path's product terms are K * 2^-23 * S.  Plane outputs are compared
as hi + lo * 2^-11 with the split's own rounding added.  tests/test_conv_ref_cpu.py checks that the fp64 convolution of
fp16-rounded operands exceeds the bound somewhere at every row, so the bound would catch a lost lo plane.

Every output is written over sentinels (NaN in fp32, 0x7E01 in planes) and must come back finite; the entry point fails when
a guard byte past an output changed."""
import ctypes
import zlib

import numpy as np
import pytest

from gtsfm_b200 import _lib
from oracle import conv_ref as cr

pytestmark = pytest.mark.gpu

PLANE_SENTINEL = 0x7E01
B2_ERR_ARG = -2

# name: (H, W, Cin, Cout, dilation, pool, relu, outputs: "planes" | "fp32" | "both")
CASES = {
    # SuperPoint (sp_conv3x3_tc, which launches through conv_ps_run): every layer writes planes, conv4b planes and fp32
    "sp_conv1b": (61, 45, 64, 64, 1, 1, 1, "planes"),
    "sp_conv2a": (300, 200, 64, 64, 1, 0, 1, "planes"),  # 475 tiles on at most 132 CTAs
    "sp_conv3a": (33, 17, 64, 128, 1, 0, 1, "planes"),
    "sp_conv3b": (31, 23, 128, 128, 1, 1, 1, "planes"),
    "sp_conv4a": (15, 20, 128, 128, 1, 0, 1, "planes"),
    "sp_conv4b": (60, 80, 128, 128, 1, 0, 1, "both"),
    "sp_convPa": (15, 20, 128, 256, 1, 0, 1, "planes"),
    "sp_convDa": (3, 5, 128, 256, 1, 0, 1, "planes"),
    # NetVLAD (nv_conv)
    "nv_conv1_2": (16, 16, 64, 64, 1, 1, 1, "planes"),
    "nv_conv2_1": (8, 8, 64, 128, 1, 0, 1, "planes"),
    "nv_conv2_2": (9, 7, 128, 128, 1, 1, 1, "planes"),
    "nv_conv3_1": (4, 4, 128, 256, 1, 0, 1, "planes"),
    "nv_conv3_2": (17, 9, 256, 256, 1, 0, 1, "planes"),
    "nv_conv3_3": (5, 3, 256, 256, 1, 1, 1, "planes"),
    "nv_conv4_1": (2, 2, 256, 512, 1, 0, 1, "planes"),
    "nv_conv4_2": (19, 11, 512, 512, 1, 0, 1, "planes"),
    "nv_conv4_3": (2, 2, 512, 512, 1, 1, 1, "planes"),
    "nv_conv5_1": (1, 1, 512, 512, 1, 0, 1, "planes"),
    "nv_conv5_2": (29, 1, 512, 512, 1, 0, 1, "planes"),
    "nv_conv5_3": (1, 37, 512, 512, 1, 0, 0, "fp32"),  # no ReLU: the last layer before the NetVLAD pooling
    # D2-Net (d2_conv): conv4_x on the dilated instance
    "d2_conv1_2": (8, 8, 64, 64, 1, 1, 1, "planes"),
    "d2_conv2_2": (3, 5, 128, 128, 1, 1, 1, "planes"),
    "d2_conv3_3": (2, 2, 256, 256, 1, 0, 1, "fp32"),
    "d2_conv4_1": (1, 1, 256, 512, 2, 0, 1, "planes"),
    "d2_conv4_2": (23, 12, 512, 512, 2, 0, 1, "planes"),
    "d2_conv4_3": (17, 10, 512, 512, 2, 0, 1, "fp32"),
    # fp32 layers at sizes that are not multiples of the tile, both dilations, with and without ReLU
    "dil2_37x29_256_512": (37, 29, 256, 512, 2, 0, 1, "fp32"),
    "dil2_13x21_512_512": (13, 21, 512, 512, 2, 0, 1, "fp32"),
    "dil2_5x3_64_128_linear": (5, 3, 64, 128, 2, 0, 0, "fp32"),
    "dil2_70x45_128_64_linear": (70, 45, 128, 64, 2, 0, 0, "fp32"),
    "dil1_37x29_256_128": (37, 29, 256, 128, 1, 0, 1, "fp32"),
}


def data(name):
    """Post-ReLU N(0, 1) activations, He-scaled weights, small biases (the statistics of a trained VGG-style layer)."""
    H, W, cin, cout = CASES[name][:4] if name in CASES else name
    rng = np.random.default_rng(zlib.crc32(str(name).encode()))
    x = np.maximum(rng.standard_normal((H, W, cin)), 0).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b = (0.05 * rng.standard_normal(cout)).astype(np.float32)
    return x, w, b


def _call(ctx, x, w, b, *, path=1, dil=1, pool=0, relu=1, ctas=0, fp32=True, planes=False):
    """One b2_debug_conv_host call: (status, fp32 output or None, hi, lo or None), outputs starting as sentinels."""
    H, W, cin = x.shape
    cout = w.shape[0]
    oh, ow = (H // 2, W // 2) if pool else (H, W)
    out = np.full((oh, ow, cout), np.nan, np.float32) if fp32 else None
    hi = np.full((oh, ow, cout), PLANE_SENTINEL, np.uint16) if planes else None
    lo = np.full((oh, ow, cout), PLANE_SENTINEL, np.uint16) if planes else None
    layer = _lib.ConvLayer(path, dil, int(pool), int(relu), ctas, H, W, cin, cout, _lib.ptr(x).value, _lib.ptr(w).value, _lib.ptr(b).value,
                           _lib.ptr(out).value, _lib.ptr(hi).value, _lib.ptr(lo).value)
    rc = ctx.lib.b2_debug_conv_host(ctx.handle, ctypes.byref(layer))
    return rc, out, hi, lo


def _run(ctx, x, w, b, **kw):
    rc, out, hi, lo = _call(ctx, x, w, b, **kw)
    ctx.check(rc, "b2_debug_conv_host")
    return out, hi, lo


def _bits(a):
    return None if a is None else a.view(np.uint32 if a.dtype == np.float32 else np.uint16)


def _same(r, s):
    return all((a is None and c is None) or np.array_equal(_bits(a), _bits(c)) for a, c in zip(r, s))


def _check(name, got, hi, lo, want, bound):
    """|got - want| <= bound element-wise for the fp32 output and for the planes' value; planes = split(fp32) when both.
    Returns the largest err / bound."""
    worst = 0.0
    if got is not None:
        assert np.isfinite(got).all(), f"{name}: an fp32 output element was not written"
        err = np.abs(got - want)
        worst = float((err / bound).max())
        assert (err <= bound).all(), (name, float(err.max()), worst)
    if hi is not None:
        v = cr.join_planes(hi, lo)
        assert np.isfinite(v).all(), f"{name}: a plane element was not written"
        pb = bound + cr.plane_error(np.abs(want) + bound)
        err = np.abs(v - want)
        worst = max(worst, float((err / pb).max()))
        assert (err <= pb).all(), (name, float(err.max()), float((err / pb).max()))
        if got is not None:
            want_hi, want_lo = cr.split_planes(got)
            assert np.array_equal(hi, want_hi) and np.array_equal(lo, want_lo), f"{name}: planes differ from the split of the fp32 output"
    return worst


@pytest.mark.parametrize("name", list(CASES))
def test_layer_matches_fp64(b200_ctx, name):
    H, W, cin, cout, dil, pool, relu, outs = CASES[name]
    x, w, b = data(name)
    kw = dict(dil=dil, pool=pool, relu=relu, fp32=outs != "planes", planes=outs != "fp32")
    first = _run(b200_ctx, x, w, b, **kw)
    second = _run(b200_ctx, x, w, b, **kw)
    assert _same(first, second), "two runs differ"
    want = cr.conv64(x, w, b, dilation=dil, pool=pool, relu=relu)
    bound = cr.bound(x, w, b, dilation=dil, pool=pool)
    print(f"err/bound {name}: {_check(name, *first, want, bound):.4f}")


# ---- schedule invariance ------------------------------------------------------------------------------------------------------
# name: (H, W, Cin, Cout, pool).  "resident": Cin = 64, the weights loaded once per CTA, 13 x 17 = 221 tiles; "reload": Cin = 256,
# the weights reloaded per (tile, chunk), 4 x 5 = 20 tiles of 8 channel blocks
SCHEDULES = {"resident": (201, 131, 64, 64, 1), "reload": (63, 37, 256, 512, 0)}


@pytest.mark.parametrize("dil", [1, 2])
@pytest.mark.parametrize("kind", list(SCHEDULES))
def test_grid_does_not_change_the_result(b200_ctx, kind, dil):
    """A tile's accumulation order does not depend on which CTA computes it: the production grid, one CTA per channel block
    walking every tile (its mbarrier phases wrap many times), an uneven 7 per block, and more CTAs than tiles (the idle ones
    must write nothing) give the same bits."""
    H, W, cin, cout, pool = SCHEDULES[kind]
    nblk, tiles = cout // 64, -(-H // 16) * -(-W // 8)
    x, w, b = data((H, W, cin, cout))
    runs = {g: _run(b200_ctx, x, w, b, dil=dil, pool=pool, ctas=g, planes=True) for g in (0, nblk, 7 * nblk, (tiles + 3) * nblk)}
    want = cr.conv64(x, w, b, dilation=dil, pool=pool)
    print(f"err/bound grid {kind} d{dil}: {_check(kind, *runs[0], want, cr.bound(x, w, b, dilation=dil, pool=pool)):.4f}")
    for g, r in runs.items():
        assert _same(r, runs[0]), f"ctas = {g} differs from the production grid"


# ---- outputs ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pool", [0, 1])
def test_planes_only_equal_the_split_of_fp32_only(b200_ctx, pool):
    x, w, b = data((33, 19, 128, 128))
    f32, _, _ = _run(b200_ctx, x, w, b, pool=pool)
    _, hi, lo = _run(b200_ctx, x, w, b, pool=pool, fp32=False, planes=True)
    both = _run(b200_ctx, x, w, b, pool=pool, planes=True)
    want_hi, want_lo = cr.split_planes(f32)
    assert np.array_equal(hi, want_hi) and np.array_equal(lo, want_lo)
    assert _same(both, (f32, hi, lo))


@pytest.mark.parametrize("H,W", [(17, 9), (33, 23), (3, 3), (16, 8), (2, 17)])
def test_pool_writes_nothing_at_row_oh_or_column_ow(b200_ctx, H, W):
    """Odd sizes put pixels of the dropped last row / column in a tile (at 17 x 9 they start a tile of their own): their
    would-be window must not be written.  Row OH lies past the output (the guard); column OW of row r is column 0 of row
    r + 1, where a stray write races the right value (the bound, and two runs agreeing)."""
    x, w, b = data((H, W, 64, 128))
    first = _run(b200_ctx, x, w, b, pool=1, planes=True)
    assert _same(first, _run(b200_ctx, x, w, b, pool=1, planes=True))
    _check(f"pool {H}x{W}", *first, cr.conv64(x, w, b, pool=True), cr.bound(x, w, b, pool=True))


@pytest.mark.parametrize("pool", [0, 1])
def test_saturated_planes_and_unclamped_fp32(b200_ctx, pool):
    """Outputs beyond fp16's +-65504: the fp32 output keeps the value, the planes are the clamped split (hi = +-65504, lo = 0)."""
    rng = np.random.default_rng(31 + pool)
    x = rng.standard_normal((21, 13, 64)).astype(np.float32) * np.float32(300.0)
    w = (rng.standard_normal((128, 64, 3, 3)) * np.sqrt(2.0 / 576) * 300.0).astype(np.float32)
    b = rng.standard_normal(128).astype(np.float32)
    got, hi, lo = _run(b200_ctx, x, w, b, pool=pool, relu=0, planes=True)
    want = cr.conv64(x, w, b, pool=pool, relu=False)
    bound = cr.bound(x, w, b, pool=pool)
    assert (got > 2 * 65504).any() and (got < -2 * 65504).any()
    assert (np.abs(got - want) <= bound).all()
    assert (hi[got > 65504] == 0x7BFF).all() and (hi[got < -65504] == 0xFBFF).all() and (lo[np.abs(got) > 65504] == 0).all()
    want_hi, want_lo = cr.split_planes(got)
    assert np.array_equal(hi, want_hi) and np.array_equal(lo, want_lo)


# ---- the SIMT path (SuperPoint under force_simt) ----------------------------------------------------------------------------
# name: (H, W, Cin, Cout, pool), SuperPoint's layer kinds; 8 x 16 is the SIMT kernel's tile
SIMT_CASES = {
    "sp_conv1b": (33, 21, 64, 64, 1),
    "sp_conv2a": (24, 16, 64, 64, 0),
    "sp_conv3a": (19, 13, 64, 128, 0),
    "sp_conv3b": (17, 11, 128, 128, 1),
    "sp_conv4b": (15, 20, 128, 128, 0),
    "sp_convPa": (7, 9, 128, 256, 0),
    "sp_convDa": (1, 3, 128, 256, 0),
}


@pytest.mark.parametrize("name", list(SIMT_CASES))
def test_simt_matches_fp64_and_wgmma(b200_ctx, name):
    H, W, cin, cout, pool = SIMT_CASES[name]
    x, w, b = data((H, W, cin, cout))
    simt, _, _ = _run(b200_ctx, x, w, b, path=0, pool=pool)
    tc, _, _ = _run(b200_ctx, x, w, b, path=1, pool=pool)
    want = cr.conv64(x, w, b, pool=pool)
    b0, b1 = cr.bound(x, w, b, pool=pool, path=0), cr.bound(x, w, b, pool=pool, path=1)
    print(f"err/bound simt {name}: {_check(name, simt, None, None, want, b0):.4f}")
    assert (np.abs(simt.astype(np.float64) - tc) <= b0 + b1).all()


# ---- refusals ---------------------------------------------------------------------------------------------------------------
# name: (overrides of a 6 x 6, 64 -> 64 wgmma layer with an fp32 output, the function that refuses it)
REFUSALS = {
    "simt_no_relu": (dict(path=0, relu=0), "b2_debug_conv_host"),
    "simt_dilation_2": (dict(path=0, dil=2), "b2_debug_conv_host"),
    "simt_cin_12": (dict(path=0, cin=12), "b2_debug_conv_host"),
    "simt_cout_96": (dict(path=0, cout=96), "b2_debug_conv_host"),
    "simt_planes": (dict(path=0, planes=True), "b2_debug_conv_host"),
    "simt_ctas": (dict(path=0, ctas=1), "b2_debug_conv_host"),
    "no_output": (dict(fp32=False), "b2_debug_conv_host"),
    "pool_of_one_row": (dict(H=1, pool=1), "b2_debug_conv_host"),
    "path_2": (dict(path=2), "b2_debug_conv_host"),
    "wgmma_cin_96": (dict(cin=96), "conv_ps"),
    "wgmma_cout_96": (dict(cout=96), "conv_ps"),
    "wgmma_cin_32": (dict(cin=32), "conv_ps"),
    "wgmma_dilation_3": (dict(dil=3), "conv_ps"),
    "wgmma_ctas_not_a_multiple": (dict(cout=128, ctas=3), "conv_ps"),
    "wgmma_ctas_negative": (dict(ctas=-1), "conv_ps"),
}


@pytest.mark.parametrize("name", list(REFUSALS))
def test_refusals(b200_ctx, name):
    o, who = REFUSALS[name]
    o = dict(o)
    H, cin, cout = o.pop("H", 6), o.pop("cin", 64), o.pop("cout", 64)
    rng = np.random.default_rng(12)
    x = rng.standard_normal((H, 6, cin)).astype(np.float32)
    w = rng.standard_normal((cout, cin, 3, 3)).astype(np.float32)
    b = np.zeros(cout, np.float32)
    rc, out, hi, _ = _call(b200_ctx, x, w, b, **o)
    assert rc == B2_ERR_ARG
    assert b200_ctx.lib.b2_last_error(b200_ctx.handle).decode().startswith(who + ":")
    assert out is None or np.isnan(out).all()
    assert hi is None or (hi == PLANE_SENTINEL).all()
