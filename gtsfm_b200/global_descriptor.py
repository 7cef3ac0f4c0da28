"""Global descriptor plugins: NetVLAD and MegaLoc.

NetVLAD global descriptor plugin (SURVEY.md section 8f rank 4: the retrieval front of deep_front_end.yaml:6-15).

Drop-in for gtsfm/frontend/global_descriptor/netvlad_global_descriptor.py:24-71 (`NetVLADGlobalDescriptor`, a
`GlobalDescriptorBase`): same `get_preprocessing_transforms` / `describe_batch(images (B, 3, H, W) float in [0, 1]) -> list of
(4096,) arrays` contract, model loaded lazily on first use.  The network of thirdparty/hloc/netvlad.py runs in
libgtsfm_b200.so (`b2_netvlad_describe_dev`): VGG16 convolutions on the SuperPoint wgmma convolution kernel, soft assignment
and whitening on the shared wgmma GEMM.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Optional, Union

import numpy as np

from . import _lib, weights
from .gtsfm_api import GlobalDescriptorBase

DEFAULT_CHECKPOINT = "thirdparty/hloc/weights/VGG16-NetVLAD-Pitts30K.mat"  # netvlad.py:25,79,96
DESC_DIM = 4096


class NetVLADEngine:
    def __init__(self, weights_src: Union[str, Path, dict], device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        sd = weights_src if isinstance(weights_src, dict) else (
            weights.load_netvlad_mat(weights_src) if str(weights_src).endswith(".mat") else weights.load_state_dict(weights_src))
        blob = weights.pack_netvlad(weights.load_state_dict(sd))
        self.ctx.check(self.ctx.lib.b2_netvlad_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "netvlad_set_weights")

    def describe(self, images: np.ndarray) -> np.ndarray:
        """images: (B, 3, H, W) float32 in [0, 1] host array -> (B, 4096)."""
        images = np.ascontiguousarray(images, np.float32)
        b, c, h, w = images.shape
        assert c == 3
        out = np.empty((b, DESC_DIM), np.float32)
        rc = self.ctx.lib.b2_netvlad_describe_host(self.ctx.handle, _lib.ptr(images), b, h, w, _lib.ptr(out))
        self.ctx.check(rc, "netvlad_describe_host")
        return out

    def describe_dev(self, images):
        """images: (B, 3, H, W) float32 CUDA tensor in [0, 1] -> (B, 4096) CUDA tensor."""
        import torch

        images = images.contiguous().float()
        b, c, h, w = images.shape
        assert c == 3 and images.is_cuda
        out = torch.empty((b, DESC_DIM), dtype=torch.float32, device=images.device)
        st = _lib.C.c_void_p(torch.cuda.current_stream(images.device).cuda_stream)
        rc = self.ctx.lib.b2_netvlad_describe_dev(self.ctx.handle, _lib.ptr(images), b, h, w, _lib.ptr(out), st)
        self.ctx.check(rc, "netvlad_describe_dev")
        return out


class B200NetVLADGlobalDescriptor(GlobalDescriptorBase):
    def __init__(self, weights_path: Union[str, Path, dict] = DEFAULT_CHECKPOINT, device: int = 0) -> None:
        super().__init__()
        if not isinstance(weights_path, dict) and not Path(weights_path).exists():
            raise FileNotFoundError(f"NetVLAD weights not found at {weights_path}")  # (the reference downloads them: no network here)
        self._weights = weights_path
        self._device = device
        self._engine: Optional[NetVLADEngine] = None  # lazy, like netvlad_global_descriptor.py:29-37

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_engine"] = None
        return d

    def _ensure_model_loaded(self) -> NetVLADEngine:
        if self._engine is None:
            self._engine = NetVLADEngine(self._weights, self._device)
        return self._engine

    def get_preprocessing_transforms(self):
        """netvlad_global_descriptor.py:39-51: (H, W, C) uint8 array -> (C, H, W) tensor; batch -> float32 / 255."""
        import torch

        def resize_transform(x):
            return torch.from_numpy(np.array(x, copy=True)).permute(2, 0, 1)

        def batch_transform(x):
            return x.type(torch.float32) / 255.0

        return resize_transform, batch_transform

    def describe_batch(self, images) -> List[np.ndarray]:
        eng = self._ensure_model_loaded()
        import torch

        if isinstance(images, torch.Tensor):
            if torch.cuda.is_available():
                out = eng.describe_dev(images.to(torch.device("cuda", self._device))).cpu().numpy()
            else:  # pragma: no cover - the engine itself needs a GPU
                out = eng.describe(images.numpy())
        else:
            out = eng.describe(np.asarray(images))
        return [d for d in out]


# ---- MegaLoc (gtsfm/frontend/global_descriptor/megaloc_global_descriptor.py:18-77, thirdparty/megaloc/megaloc.py) ------------------
MEGALOC_DIM = 8448
MEGALOC_SIZE = 322


class MegaLocEngine:
    """DINOv2 ViT-B/14 + SALAD + Linear(16640 -> 8448) in libgtsfm_b200.so (`b2_megaloc_*`)."""

    def __init__(self, weights_src: Union[str, Path, dict], device: int = 0, ctx: Optional[_lib.Context] = None):
        self.ctx = ctx or _lib.Context(device)
        blob = weights.pack_megaloc(weights.load_megaloc(weights_src))
        self.ctx.check(self.ctx.lib.b2_megaloc_set_weights(self.ctx.handle, _lib.ptr(blob), blob.size), "megaloc_set_weights")

    def describe(self, images: np.ndarray) -> np.ndarray:
        """images: (B, 3, H, W) float32 host array, normalised, H and W multiples of 14 -> (B, 8448)."""
        images = np.ascontiguousarray(images, np.float32)
        b, c, h, w = images.shape
        assert c == 3
        out = np.empty((b, MEGALOC_DIM), np.float32)
        self.ctx.check(self.ctx.lib.b2_megaloc_describe_host(self.ctx.handle, _lib.ptr(images), b, h, w, _lib.ptr(out)), "megaloc_describe_host")
        return out

    def describe_dev(self, images):
        """images: (B, 3, H, W) float32 CUDA tensor, normalised -> (B, 8448) CUDA tensor."""
        import torch

        images = images.contiguous().float()
        b, c, h, w = images.shape
        assert c == 3 and images.is_cuda
        out = torch.empty((b, MEGALOC_DIM), dtype=torch.float32, device=images.device)
        st = _lib.C.c_void_p(torch.cuda.current_stream(images.device).cuda_stream)
        self.ctx.check(self.ctx.lib.b2_megaloc_describe_dev(self.ctx.handle, _lib.ptr(images), b, h, w, _lib.ptr(out), st), "megaloc_describe_dev")
        return out

    @staticmethod
    def _u8_args(frames):
        import torch

        frames = [f if f.is_contiguous() else f.contiguous() for f in frames]
        h, w, c = frames[0].shape
        assert c == 3 and all(f.shape == frames[0].shape and f.dtype == torch.uint8 and f.is_cuda for f in frames)
        ptrs = (_lib.C.c_void_p * len(frames))(*[f.data_ptr() for f in frames])
        return frames, ptrs, h, w, w * 3

    def describe_u8_dev(self, frames):
        """frames: list of same-shape (H, W, 3) uint8 CUDA tensors (RGB) -> (n, 8448) CUDA tensor: the plugin's resize to
        322 x 322 and normalisation run on the device too."""
        import torch

        frames, ptrs, h, w, pitch = self._u8_args(frames)
        out = torch.empty((len(frames), MEGALOC_DIM), dtype=torch.float32, device=frames[0].device)
        st = _lib.C.c_void_p(torch.cuda.current_stream(frames[0].device).cuda_stream)
        rc = self.ctx.lib.b2_megaloc_describe_u8_dev(self.ctx.handle, ptrs, len(frames), h, w, pitch, _lib.ptr(out), st)
        self.ctx.check(rc, "megaloc_describe_u8_dev")
        return out

    def resize_u8_dev(self, frames):
        """frames as for describe_u8_dev -> (n, 3, 322, 322) uint8 CUDA tensor (the plugin's resize transform)."""
        import torch

        frames, ptrs, h, w, pitch = self._u8_args(frames)
        out = torch.empty((len(frames), 3, MEGALOC_SIZE, MEGALOC_SIZE), dtype=torch.uint8, device=frames[0].device)
        st = _lib.C.c_void_p(torch.cuda.current_stream(frames[0].device).cuda_stream)
        self.ctx.check(self.ctx.lib.b2_megaloc_resize_u8_dev(self.ctx.handle, ptrs, len(frames), h, w, pitch, _lib.ptr(out), st), "megaloc_resize_u8_dev")
        return out


class B200MegaLocGlobalDescriptor(GlobalDescriptorBase):
    """Drop-in for `MegaLocGlobalDescriptor`: the reference's own preprocessing transforms, `describe_batch` -> list of
    (8448,) float32 arrays, the model loaded lazily on first use.

    Deliberate difference: a missing checkpoint raises FileNotFoundError here, where the reference logs a warning and
    carries on with randomly initialised weights (megaloc.py:52-66), which would silently produce meaningless pairs."""

    def __init__(self, weights_path: Union[str, Path, dict] = "megaloc.torch", device: int = 0) -> None:
        super().__init__()
        if not isinstance(weights_path, dict) and not Path(weights_path).exists():
            raise FileNotFoundError(f"MegaLoc weights not found at {weights_path}")
        self._weights = weights_path
        self._device = device
        self._engine: Optional[MegaLocEngine] = None

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_engine"] = None
        return d

    def _ensure_model_loaded(self) -> MegaLocEngine:
        if self._engine is None:
            self._engine = MegaLocEngine(self._weights, self._device)
        return self._engine

    def get_preprocessing_transforms(self):
        """megaloc_global_descriptor.py:36-62: (H, W, C) uint8 array -> (C, 322, 322) uint8 tensor (antialiased resize);
        batch -> float32 / 255, ImageNet normalisation."""
        import torch
        from torchvision.transforms import v2 as transforms

        resize_transform = transforms.Compose([
            transforms.Lambda(lambda x: torch.from_numpy(x)),
            transforms.Lambda(lambda x: x.permute(2, 0, 1)),
            transforms.Resize(size=(MEGALOC_SIZE, MEGALOC_SIZE), antialias=True),
        ])
        batch_transform = transforms.Compose([
            transforms.Lambda(lambda x: x.type(torch.float32) / 255.0),
            transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]),
        ])
        return resize_transform, batch_transform

    def describe_batch(self, images) -> List[np.ndarray]:
        eng = self._ensure_model_loaded()
        import torch

        if isinstance(images, torch.Tensor):
            out = eng.describe_dev(images.to(torch.device("cuda", self._device))).cpu().numpy()
        else:
            out = eng.describe(np.asarray(images))
        return [d for d in out]
