"""GPU suite: b2_jpeg_decode_batched_dev equals np.asarray(PIL.Image.open(f).convert("RGB")) bit for bit on the generated corpus
and the committed fixtures, batches equal per-image calls, corrupt scans fail alone, and ingest_jpeg -> detect equals the
host-decoded path."""
import io

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import jpeg_ref as J

pytestmark = pytest.mark.gpu

FIXTURES = ["lund_door_DSC_0001.JPG", "lund_door_DSC_0002.JPG", "1dsfm_1216783_98f2f3e4e1_o.jpg"]


def _pil(data: bytes) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.fixture(scope="module")
def engine(b200_ctx):
    from gtsfm_b200.image_io import JpegEngine

    return JpegEngine(0, ctx=b200_ctx)


@pytest.fixture(scope="module")
def corpus():
    return J.corpus()


def test_bit_exact_on_corpus(engine, corpus):
    out = engine.decode_many([d for _, d in corpus])
    bad = [name for (name, d), t in zip(corpus, out) if not np.array_equal(t.cpu().numpy(), _pil(d))]
    assert not bad, bad
    assert min(engine.last_rounds) >= 1  # 9 = the serial chain finished an image the rounds had not synchronised


@pytest.mark.parametrize("name", FIXTURES)
def test_bit_exact_on_fixture(engine, golden_dir, name):
    d = (golden_dir / "jpeg" / name).read_bytes()
    assert np.array_equal(engine.decode(d).cpu().numpy(), _pil(d))
    assert engine.last_rounds[0] <= 8  # synchronised by the rounds, not by the serial chain


def test_large_frame_synchronises_in_the_rounds(engine):
    d = J.encode(J.content("synthetic", 3000, 4000, seed=2), "420", quality=90)
    assert np.array_equal(engine.decode(d).cpu().numpy(), _pil(d))
    assert engine.last_rounds[0] <= 8


def test_mixed_batch_equals_single_calls_and_repeats(engine, corpus, golden_dir):
    names = ["1x1-noise-420-q75", "37x53-noise-444-q95", "517x389-synthetic-L-q90", "16x16-grad-422-restart_marker_blocks1",
             "517x389-noise-422-rmr1-opt", "15x17-flat-420-q1"]
    files = [dict(corpus)[n] for n in names]
    files.insert(2, (golden_dir / "jpeg" / FIXTURES[0]).read_bytes())
    files.insert(5, (golden_dir / "jpeg" / FIXTURES[2]).read_bytes())
    single = [engine.decode(d).cpu() for d in files]
    for _ in range(2):
        batch = engine.decode_many(files)
        for s, b in zip(single, batch):
            assert torch.equal(s, b.cpu())


def test_corrupt_scans_fail_alone(engine, corpus, golden_dir):
    good = [dict(corpus)["37x53-noise-420-q95"], (golden_dir / "jpeg" / FIXTURES[2]).read_bytes()]
    src = dict(corpus)["517x389-noise-420-q90"]
    scan = J.parse(src).scan_offset
    # the scan cut short, with the EOI kept so the header parse accepts it: too few MCUs
    truncated = src[:scan + (len(src) - scan) // 2] + b"\xff\xd9"
    # a marker planted in the middle of the scan ends it early
    planted = bytearray(src)
    mid = scan + (len(src) - scan) // 3
    planted[mid:mid + 2] = b"\xff\xd9"
    # flipped bytes inside the scan: either refused, or decoded as PIL decodes the same bytes
    flips = []
    for k in range(4):
        f = bytearray(src)
        p = scan + (len(src) - scan) * (k + 1) // 6
        f[p] = f[p] ^ 0x5A if f[p] ^ 0x5A != 0xFF else 0x11
        if f[p - 1] == 0xFF:  # keep the stuffing intact so the flip stays inside the entropy-coded data
            f[p] = 0x00
        flips.append(bytes(f))
    files = [good[0], truncated, bytes(planted), good[1]] + flips
    out = engine.decode_many(files, return_errors=True)
    assert np.array_equal(out[0].cpu().numpy(), _pil(good[0]))
    assert np.array_equal(out[3].cpu().numpy(), _pil(good[1]))
    assert isinstance(out[1], ValueError) and isinstance(out[2], ValueError)
    for f, o in zip(flips, out[4:]):
        if not isinstance(o, ValueError):
            assert np.array_equal(o.cpu().numpy(), _pil(f))
    assert sum(isinstance(o, ValueError) for o in out[4:]) >= 1
    with pytest.raises(ValueError):
        engine.decode_many([good[0], truncated])
    # unsupported files are refused before anything is uploaded
    for name, d in J.unsupported_cases():
        assert isinstance(engine.decode_many([d], return_errors=True)[0], ValueError), name


def test_ingest_jpeg_then_detect_equals_host_decode(b200_ctx, golden_dir):
    from gtsfm_b200 import synthetic as syn
    from gtsfm_b200.pipeline import DeviceFrontEnd

    fe = DeviceFrontEnd(syn.superpoint_state_dict(0), ctx=b200_ctx)
    datas = [(golden_dir / "jpeg" / n).read_bytes() for n in FIXTURES[:2]]
    frames = fe.ingest_jpeg(datas)
    for d, f in zip(datas, frames):
        host = torch.from_numpy(_pil(d).copy()).to(fe.device)
        ref = fe.ingest(host)
        assert torch.equal(f, ref)
        a, b = fe.detect(f), fe.detect(ref)
        assert torch.equal(a.kp, b.kp) and torch.equal(a.score, b.score) and torch.equal(a.desc, b.desc)
        assert len(a.kp) > 0


def test_load_image_matches_reference_semantics(golden_dir):
    from PIL.ExifTags import GPSTAGS, TAGS

    from gtsfm_b200 import image_io

    for name in FIXTURES:
        path = golden_dir / "jpeg" / name
        img = image_io.load_image(path)
        pil = Image.open(path)
        raw = pil._getexif()
        exif = None if raw is None else {TAGS.get(k, GPSTAGS.get(k, k)) if (k in TAGS or k in GPSTAGS) else k: v
                                         for k, v in raw.items()}
        assert np.array_equal(img.value_array, np.asarray(pil.convert("RGB")))
        assert img.exif_data == exif and img.exif_data is not None
        assert img.file_name == name
