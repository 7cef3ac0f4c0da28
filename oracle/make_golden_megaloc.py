"""Goldens for the MegaLoc global descriptor: tests/golden/megaloc.npz, from the reference's own MegaLocModel forward.

The model is assembled offline from unmodified reference code (thirdparty/megaloc/megaloc.py): `torch.hub.load` is given
DINOv2's own DinoVisionTransformer (vit_base, patch 14, img_size 518, init_values 1.0, block_chunks 0 - hub's dinov2_vitb14 in
state-dict names and forward; shipped in thirdparty/vggt/vggt/layers/vision_transformer.py), the checkpoint download is made
to fail (the model then keeps its init, which `load_state_dict(megaloc_state_dict(seed), strict=True)` replaces), and dask
(imported only by gtsfm.utils.logger) is stubbed.  The oracle restatement (oracle/megaloc_ref.py) is checked against the
module before anything is written.

Recorded per case: the module's fp32 descriptors, the largest |fp32 - fp64| of the same module in double (the spread that
sets the GPU bar), and for one image the backbone's final-LN cls token and every 16th patch token.  The input frames are
rebuilt from their seeds by the tests (only their byte sums are stored), which keeps the file small.  `python oracle/make_golden_megaloc.py`
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from gtsfm_b200 import synthetic as syn  # noqa: E402
from oracle import megaloc_ref, ref_modules  # noqa: E402

OUT = ROOT / "tests" / "golden"
SEED = 5


def reference_model():
    class _Stub(types.ModuleType):
        def __getattr__(self, n):
            if n.startswith("__"):
                raise AttributeError(n)
            return type(n, (), {"__init__": lambda self, *a, **k: None})

    for name in ("dask", "dask.distributed", "distributed"):
        sys.modules.setdefault(name, _Stub(name))
    ref = str(ref_modules.REF)
    for p in (ref, ref + "/thirdparty/vggt"):
        if p not in sys.path:
            sys.path.insert(0, p)
    from vggt.layers.vision_transformer import vit_base

    def _offline(*a, **k):
        raise RuntimeError("offline")

    hub_load, hub_url = torch.hub.load, torch.hub.load_state_dict_from_url
    torch.hub.load = lambda *a, **k: vit_base(patch_size=14, img_size=518, init_values=1.0, block_chunks=0)
    torch.hub.load_state_dict_from_url = _offline
    try:
        from thirdparty.megaloc.megaloc import MegaLocModel

        m = MegaLocModel().eval()
    finally:
        torch.hub.load, torch.hub.load_state_dict_from_url = hub_load, hub_url
    m.load_state_dict({k: torch.from_numpy(v) for k, v in syn.megaloc_state_dict(SEED).items()}, strict=True)
    return m


def frames_322():
    """The plugin's resize transform (torchvision) on the seeded frames of `megaloc_ref.GOLDEN_FRAMES`.  The frames are not stored:
    the tests rebuild them with `megaloc_ref.golden_frames_u8`, which must give the same bytes."""
    from torchvision.transforms import v2 as T

    rs = T.Resize(size=(322, 322), antialias=True)
    u8 = np.stack([rs(torch.from_numpy(syn.synthetic_frame(i, h, w)).permute(2, 0, 1)).numpy() for i, h, w in megaloc_ref.GOLDEN_FRAMES])
    assert np.array_equal(u8, megaloc_ref.golden_frames_u8()), "the NumPy resize restatement differs from torchvision"
    return u8


def shifted_322():
    """Frame 0's scene seen 14 px further right: a shifted view of the same scene."""
    big = syn.synthetic_frame(60, 480, 640)
    return megaloc_ref.normalise(megaloc_ref.resize_u8(np.ascontiguousarray(np.pad(big[:, 14:], ((0, 0), (0, 14), (0, 0)), mode="edge"))))


def other_image(seed, h, w):
    im = syn.synthetic_frame(seed, h, w).transpose(2, 0, 1)
    return megaloc_ref.normalise(np.ascontiguousarray(im))


def main():
    assert ref_modules.available(), "the reference checkout is required"
    torch.set_num_threads(16)
    m = reference_model()
    md = reference_model().double()
    sd = syn.megaloc_state_dict(SEED)
    out = {"versions": np.array(str(dict(torch=torch.__version__, numpy=np.__version__)))}

    def run(x):
        with torch.no_grad():
            y = m(torch.from_numpy(x)).numpy()
            y64 = md(torch.from_numpy(x).double()).numpy()
        mine = megaloc_ref.megaloc_forward(sd, x)
        err = float(np.abs(mine - y).max())
        assert err < 1e-5, f"restatement differs from the module: {err}"
        return y, float(np.abs(y.astype(np.float64) - y64).max()), err

    u8 = frames_322()
    x = megaloc_ref.normalise(u8)
    out["u8_322_sum"] = u8.reshape(len(u8), -1).sum(1, dtype=np.int64)
    y, spread, err = run(x)
    out["desc_322"], out["spread_322"] = y, np.float64(spread)
    print("322 frames: spread fp32/fp64", spread, "restatement", err)
    cos = y @ y.T
    out["cos_322"] = cos
    diffs = [np.abs(y[i] - y[j]).max() for i in range(len(y)) for j in range(i + 1, len(y))]
    out["min_pair_maxdiff"] = np.float64(min(diffs))
    print("cosines\n", np.round(cos, 4), "\nsmallest max|d_i - d_j|", min(diffs))
    # a batch with a repeated frame
    yb, sb, _ = run(x[[0, 2, 0]])
    out["desc_batch_0_2_0"], out["spread_batch"] = yb, np.float64(sb)
    # a shifted view of frame 0 must be nearer to frame 0 than any other frame is
    ys, _, _ = run(shifted_322()[None])
    out["desc_shift_0"] = ys
    print("shifted view cos to frames", np.round(ys @ y.T, 4))
    assert (ys @ y.T)[0, 0] > max((ys @ y.T)[0, 1:]), "the shifted view is not nearest to its frame"
    # backbone tokens of frame 0 (fault localisation)
    with torch.no_grad():
        tok = megaloc_ref.backbone(megaloc_ref.tensors(sd), torch.from_numpy(x[:1]))[0].numpy()
        tok_mod = m.backbone.model.forward_features(torch.from_numpy(x[:1]))
    assert np.abs(tok[0] - tok_mod["x_norm_clstoken"][0].numpy()).max() < 1e-4
    assert np.abs(tok[1:] - tok_mod["x_norm_patchtokens"][0].numpy()).max() < 1e-4
    out["tokens_0_rows"] = megaloc_ref.GOLDEN_TOKEN_ROWS
    out["tokens_0"] = tok[megaloc_ref.GOLDEN_TOKEN_ROWS]
    # a non-square size (interpolated position table) and 518 x 518 (the table as is)
    for name, (seed, h, w) in (("224x308", (70, 224, 308)), ("518", (71, 518, 518))):
        xi = other_image(seed, h, w)[None]
        yi, si, _ = run(xi)
        out[f"desc_{name}"], out[f"spread_{name}"] = yi, np.float64(si)
        print(name, "spread", si)
    OUT.mkdir(parents=True, exist_ok=True)
    np.savez_compressed(OUT / "megaloc.npz", **out)
    print("wrote", OUT / "megaloc.npz", (OUT / "megaloc.npz").stat().st_size)


if __name__ == "__main__":
    main()
