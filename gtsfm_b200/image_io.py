"""JPEG decode on the device: file bytes -> device RGB frames equal to what the reference's loader gets from PIL.

The reference opens every frame with `np.asarray(PIL.Image.open(f).convert("RGB"))` (gtsfm/utils/io.py:39-72); the pixels of
a baseline JPEG come from libjpeg-turbo's default path, which `b2_jpeg_decode_batched_dev` restates bit for bit on the GPU
(include/gtsfm_b200.h).  There is no CPU fallback: a file outside the decoder's scope (progressive, CMYK, 12-bit, other
sampling factors ...) raises ValueError naming the feature, and a caller that has to accept such files opens them with PIL.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import List, Optional, Sequence, Tuple, Union

import torch

from . import _lib
from .gtsfm_api import Image

MAX_BATCH = 256  # b2_jpeg_decode_batched_dev


def _status_text(code: int) -> str:
    return _lib.load().b2_jpeg_status_string(int(code)).decode()


def jpeg_info(data: bytes) -> Tuple[int, int, int]:
    """(height, width, components) from the header alone; ValueError for a file the device decoder does not accept."""
    lib = _lib.load()
    h, w, c = C.c_int(0), C.c_int(0), C.c_int(0)
    rc = lib.b2_jpeg_info_host(C.c_char_p(data), len(data), C.byref(h), C.byref(w), C.byref(c))
    if rc != 0:
        raise ValueError(f"JPEG not decodable on the device ({rc}): {_status_text(rc)}")
    return h.value, w.value, c.value


class JpegEngine:
    """Batched device decoder.  The context is created on first use and never pickled."""

    def __init__(self, device: int = 0, ctx: Optional[_lib.Context] = None):
        self._device = device
        self._ctx = ctx
        self.last_rounds: List[int] = []  # synchronisation rounds per image of the last decode_many

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_ctx"] = None
        return st

    def _ensure_ctx(self) -> _lib.Context:
        if self._ctx is None:
            self._ctx = _lib.Context(self._device)
        return self._ctx

    @staticmethod
    def info(data: bytes) -> Tuple[int, int, int]:
        return jpeg_info(data)

    def decode(self, data: bytes) -> torch.Tensor:
        return self.decode_many([data])[0]

    def decode_many(self, datas: Sequence[bytes], return_errors: bool = False) -> List[Union[torch.Tensor, ValueError]]:
        """Device uint8 (H, W, 3) tensors, one per file, on the current stream of the engine's device.  A file that cannot be
        decoded raises ValueError, or with return_errors=True takes a ValueError in its place while the others decode."""
        ctx = self._ensure_ctx()
        dev = torch.device("cuda", ctx.device)
        out: List[Union[torch.Tensor, ValueError]] = []
        self.last_rounds = []
        for b0 in range(0, len(datas), MAX_BATCH):
            chunk = [bytes(d) for d in datas[b0:b0 + MAX_BATCH]]
            shapes = []
            for d in chunk:
                try:
                    shapes.append(jpeg_info(d)[:2])
                except ValueError as e:
                    shapes.append(e)
            tensors = [torch.empty((s[0], s[1], 3), dtype=torch.uint8, device=dev) if isinstance(s, tuple) else None for s in shapes]
            arr = (_lib.JpegImage * len(chunk))()
            for i, (d, t) in enumerate(zip(chunk, tensors)):
                arr[i].data = C.cast(C.c_char_p(d), C.c_void_p)
                arr[i].size = len(d)
                arr[i].out = t.data_ptr() if t is not None else None
                arr[i].out_pitch = t.shape[1] * 3 if t is not None else 0
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            ctx.check(ctx.lib.b2_jpeg_decode_batched_dev(ctx.handle, arr, len(chunk), stream), "jpeg_decode_batched_dev")
            for i, t in enumerate(tensors):
                rc = arr[i].out_status
                self.last_rounds.append(int(arr[i].out_rounds))
                if rc == 0 and t is not None:
                    out.append(t)
                    continue
                err = shapes[i] if isinstance(shapes[i], ValueError) else \
                    ValueError(f"JPEG not decodable on the device ({rc}): {_status_text(rc)}")
                if not return_errors:
                    raise ValueError(f"image {b0 + i}: {err}")
                out.append(err)
        return out


def read_exif(img_path: Union[str, Path]):
    """The reference's EXIF dictionary (gtsfm/utils/io.py:54-68) from PIL's lazy header read: no pixels are decoded."""
    from PIL import Image as PILImage
    from PIL.ExifTags import GPSTAGS, TAGS

    with PILImage.open(str(img_path)) as original_image:
        exif_data = original_image._getexif() if hasattr(original_image, "_getexif") else None
    if exif_data is None:
        return None
    parsed = {}
    for tag_id, value in exif_data.items():
        if tag_id in TAGS:
            name = TAGS.get(tag_id)
        elif tag_id in GPSTAGS:
            name = GPSTAGS.get(tag_id)
        else:
            name = tag_id
        parsed[name] = value
    return parsed


_default_engine: Optional[JpegEngine] = None


def load_image(img_path: Union[str, Path], engine: Optional[JpegEngine] = None) -> Image:
    """Drop-in for gtsfm/utils/io.py:39-72 load_image on JPEG files: the same host value_array (H x W x 3 uint8, decoded on
    the GPU) and the same EXIF dictionary; EXIF orientation is not applied, as the reference does not apply it."""
    global _default_engine
    if engine is None:
        if _default_engine is None:
            _default_engine = JpegEngine()
        engine = _default_engine
    data = Path(img_path).read_bytes()
    rgb = engine.decode(data).cpu().numpy()
    return Image(value_array=rgb, exif_data=read_exif(img_path), file_name=Path(img_path).name)
