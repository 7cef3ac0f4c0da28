"""CPU suite: the JPEG oracle restates PIL's decode bit for bit, the subsequence-synchronisation model gives the sequential
decode's coefficients, and the library's header parse (b2_jpeg_info_host, no GPU) accepts and refuses what it should."""
import io

import numpy as np
import pytest
from PIL import Image

from oracle import jpeg_ref as J

FIXTURES = ["lund_door_DSC_0001.JPG", "lund_door_DSC_0002.JPG", "1dsfm_1216783_98f2f3e4e1_o.jpg"]


def _pil(data: bytes) -> np.ndarray:
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


@pytest.fixture(scope="module")
def corpus():
    return J.corpus()


def test_oracle_equals_pil_on_corpus(corpus):
    bad = [name for name, d in corpus if not np.array_equal(J.decode(d), _pil(d))]
    assert not bad, bad


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_equals_pil_on_fixture(golden_dir, name):
    d = (golden_dir / "jpeg" / name).read_bytes()
    assert np.array_equal(J.decode(d), _pil(d))


def test_fixture_sampling(golden_dir):
    lund = J.parse((golden_dir / "jpeg" / FIXTURES[0]).read_bytes())
    assert (lund.comps[0].h, lund.comps[0].v) == (1, 2) and (lund.height, lund.width) == (1936, 1296)
    ds = J.parse((golden_dir / "jpeg" / FIXTURES[2]).read_bytes())
    assert (ds.comps[0].h, ds.comps[0].v) == (2, 2)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", ["37x53-noise-420-q100", "37x53-noise-422-restart_marker_blocks3", "37x53-grad-444-q1",
                                  "15x17-noise-L-restart_marker_blocks1", "37x53-noise-444-restart_marker_rows1"])
def test_sync_model_matches_sequential(corpus, name):
    d = dict(corpus)[name]
    _, ref = J.decode_coefficients(d)
    stream, _ = J.unstuff(d, J.parse(d).scan_offset)
    nbits = 8 * len(stream)
    divisor = next(k for k in (7, 5, 3, 2, 1) if nbits % k == 0)
    # incl. a length that divides the scan and ones longer than it, and chunks of 1, 4 and the device's 256 subsequences
    for sub in (33, 100, 1024, nbits // divisor, nbits, 4 * nbits):
        for chunk in (1, 4, J.SYNC_CHUNK):
            st = {}
            got, rounds = J.sync_decode(d, sub, chunk, J.SYNC_ROUNDS, st)
            assert _same(ref, got), (name, sub, chunk)
            assert 1 <= rounds <= J.SYNC_ROUNDS + 1 and (st["serial"] > 0) == (rounds > J.SYNC_ROUNDS)


def test_sync_model_converges_on_photo_at_device_parameters(golden_dir):
    """The 1DSfM frame (h2v2, 2200 subsequences of 1024 bits, 9 chunks) synchronises in the rounds: no serial chain, and the
    chunk pass decodes each subsequence only a few times."""
    d = (golden_dir / "jpeg" / FIXTURES[2]).read_bytes()
    _, ref = J.decode_coefficients(d)
    st = {}
    got, rounds = J.sync_decode(d, stats=st)
    assert _same(ref, got)
    assert rounds <= 3 and st["serial"] == 0, (rounds, st)
    n_sub = -(-8 * len(J.unstuff(d, J.parse(d).scan_offset)[0]) // J.SYNC_SUB_BITS)
    assert st["chunk"] < 4 * n_sub and st["rounds"] < n_sub // 10, st


def test_sync_model_serial_fallback(corpus):
    """With one-subsequence chunks and a single round the rounds cannot settle a noise scan: the serial chain finishes it
    and the coefficients are still the sequential decode's."""
    d = dict(corpus)["37x53-noise-444-q100"]
    _, ref = J.decode_coefficients(d)
    st = {}
    got, rounds = J.sync_decode(d, 64, 1, 1, st)
    assert rounds == 2 and st["serial"] > 0
    assert _same(ref, got)


def test_unstuff_removes_stuffing_and_markers(corpus):
    d = dict(corpus)["37x53-noise-420-restart_marker_blocks1"]
    stream, rst = J.unstuff(d, J.parse(d).scan_offset)
    g = J.geometry(J.parse(d))
    assert len(rst) == g.mcux * g.mcuy - 1  # one marker between consecutive MCUs
    assert rst == sorted(rst) and len(stream) < len(d)


def _lib():
    from gtsfm_b200 import _lib

    return _lib.load()


def _info(data: bytes):
    import ctypes as C

    h, w, c = C.c_int(-1), C.c_int(-1), C.c_int(-1)
    rc = _lib().b2_jpeg_info_host(C.c_char_p(data), len(data), C.byref(h), C.byref(w), C.byref(c))
    return rc, (h.value, w.value, c.value)


def test_info_accepts_corpus(corpus, golden_dir):
    files = list(corpus) + [(n, (golden_dir / "jpeg" / n).read_bytes()) for n in FIXTURES]
    for name, d in files:
        rc, hwc = _info(d)
        im = Image.open(io.BytesIO(d))
        assert rc == 0, (name, rc)
        assert hwc == (im.height, im.width, 1 if im.mode == "L" else 3), name


def test_info_refuses_unsupported():
    from gtsfm_b200 import image_io

    for name, d in J.unsupported_cases():
        rc, _ = _info(d)
        assert rc < 0, name
        with pytest.raises(ValueError):
            image_io.jpeg_info(d)
    d = J.unsupported_cases()[0][1]
    with pytest.raises(ValueError, match="progressive"):
        image_io.jpeg_info(d)


def test_info_refuses_truncation_everywhere(golden_dir):
    d = (golden_dir / "jpeg" / FIXTURES[2]).read_bytes()
    rng = np.random.default_rng(0)
    for cut in sorted(set([0, 1, 2, 3, 20, 200, 2000, len(d) // 3, len(d) - 3, len(d) - 2, len(d) - 1]
                          + rng.integers(4, len(d) - 1, 10).tolist())):
        rc, _ = _info(d[:cut])
        assert rc < 0, cut


def test_info_limits_and_status_strings():
    lib = _lib()
    assert b"progressive" in lib.b2_jpeg_status_string(-11)
    assert b"CMYK" in lib.b2_jpeg_status_string(-15)
    # a frame header announcing 20000 x 20000 pixels is beyond the limits (-2), not decoded
    d = bytearray(J.encode(J.content("flat", 16, 16), "444", quality=75))
    p = d.find(b"\xff\xc0")
    d[p + 5:p + 9] = (20000).to_bytes(2, "big") + (20000).to_bytes(2, "big")
    assert _info(bytes(d))[0] == -2


def test_engine_pickles_without_a_device():
    import pickle

    from gtsfm_b200.image_io import JpegEngine

    e = pickle.loads(pickle.dumps(JpegEngine(0)))
    assert e._ctx is None
