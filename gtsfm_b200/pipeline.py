"""Device-resident batched front-end: detect -> top-k -> describe -> match -> verify with every tensor kept in HBM.

This is the L2 seam of SURVEY.md §8b (`CorrespondenceGeneratorBase.generate_correspondences`): instead of one Dask task
per image and per pair, each pickling ~5 MB of features (det_desc_correspondence_generator.py:65-85), one process per
GPU walks its shard of the visibility graph and only small results (match index arrays, E / R / t) leave the device.
PyTorch is used for device buffers and the stream only; all arithmetic is libgtsfm_b200.so through the `*_dev` C ABI.

Besides its own library context, a front end runs "lanes": more contexts, each with its own work buffers, stream and (for
the roles driven from host threads) one host thread, so that independent images or pairs overlap on the GPU.  `detect_many`
uses DETECT_LANES of them, `match_superglue_many` SG_LANES and verification one.  Every lane is configured like the front
end's context: its recorded options are replayed onto the lane before the lane loads its model's weights.
"""
from __future__ import annotations

import contextlib
import itertools
import os
import threading
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib, weights
from .detector_descriptor import KEYPOINT_THRESHOLD, NMS_RADIUS, REMOVE_BORDERS, SuperPointEngine
from .verifier import DEFAULT_SEED, E_MAX_ITERS, LMEDS_MAX_ITERS, RANSAC_SUCCESS_PROB, lmeds_params, ransac_problem


@dataclass
class DeviceFeatures:
    kp: torch.Tensor  # (k, 2) float32 (x, y), device
    score: torch.Tensor  # (k,) float32 response
    desc: torch.Tensor  # (k, D) in the detector's dtype: SuperPoint f32 x 256, SIFT u8 x 128, ORB u8 x 32, D2-Net f32 x 512
    shape: Tuple[int, int]
    scale: Optional[torch.Tensor] = None  # (k,) float32 keypoint size, for the detectors whose Keypoints carry scales (SIFT, ORB)
    # LightGlue's pair-independent layer-0 state of this image (b2_lightglue_encode_batched_dev), made on first use by
    # DeviceFrontEnd.match_batch / match_many and keyed by DeviceFrontEnd._enc_key(); freed with the features
    enc: Dict[tuple, torch.Tensor] = field(default_factory=dict, repr=False, compare=False)

    def __len__(self) -> int:
        return int(self.kp.shape[0])


SG_LANES = int(os.environ.get("B2_SG_LANES", "3"))  # concurrent SuperGlue instances used by match_superglue_many
DETECT_LANES = int(os.environ.get("B2_DETECT_LANES", "4"))  # concurrent SuperPoint instances used by detect_many
# SMs the matcher's persistent kernels leave to the concurrent RANSAC kernels.  H100 (132 SMs), 40-pair LightGlue steps:
# 99 pairs/s reserving 8, 103-107 reserving 0-4; 4 keeps k_rs_hyp_E's CTAs off the matcher's SMs at no measured cost
RESERVE_SMS_FOR_VERIFY = int(os.environ.get("B2_RESERVE_SMS", "4"))
_FRONT_END_SERIAL = itertools.count()  # one per DeviceFrontEnd: an image's LightGlue encoding is only valid for the one that made it
# model -> (weights packer, the library entry point that loads the packed weights onto a context)
_MODELS = {"superpoint": (weights.pack_superpoint, "b2_superpoint_set_weights"),
           "lightglue": (weights.pack_lightglue, "b2_lightglue_set_weights"),
           "superglue": (weights.pack_superglue, "b2_superglue_set_weights")}


@dataclass
class _Lane:
    """A library context (own work buffers), the stream its work is enqueued on and, if its role needs one, a host thread."""
    ctx: _lib.Context
    stream: Optional[torch.cuda.Stream] = None  # None: the caller's current stream (the front end's own context)
    pool: Optional[ThreadPoolExecutor] = None  # the lane's host thread, for the roles that drive lanes from threads


class DeviceFrontEnd:
    def __init__(self, superpoint_sd, lightglue_sd=None, device: int = 0, max_keypoints: int = 5000, cpu_semantics: bool = True,
                 ctx: Optional[_lib.Context] = None, superglue_sd=None, fp16_attention: bool = False):
        if not torch.cuda.is_available():
            raise _lib.B200Error("DeviceFrontEnd needs a CUDA device; there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.ctx = ctx or _lib.Context(device)
        self.lib = self.ctx.lib
        self.max_keypoints = max_keypoints
        self.prune_min = -1 if cpu_semantics else 1536
        self.fp16_attention = 1 if fp16_attention else 0  # opt-in: the reference's CUDA numerics (lightglue.py:116-121)
        self._counts = None
        self._serial = next(_FRONT_END_SERIAL)
        self._blobs = {}  # model -> packed weights, kept for the lanes that run the model
        for model, sd in (("superpoint", superpoint_sd), ("lightglue", lightglue_sd), ("superglue", superglue_sd)):
            if sd is not None:
                self._blobs[model] = _MODELS[model][0](weights.load_state_dict(sd))
                self._set_weights(self.ctx, model)
        self._lanes: Dict[str, List[_Lane]] = {"superpoint": [], "superglue": []}  # model -> its lanes, made by _role_lanes
        # verification runs on its own lane so that the (latency-bound, 16-CTA) RANSAC kernels of pair p overlap the matcher
        # kernels of pair p+1 (ctypes calls release the GIL)
        self._vlane: Optional[_Lane] = None
        self._lane_lock = threading.RLock()  # verify_async makes the verification lane from matcher callback threads

    def _set_weights(self, ctx: _lib.Context, model: str) -> None:
        blob, entry = self._blobs[model], _MODELS[model][1]
        ctx.check(getattr(self.lib, entry)(ctx.handle, _lib.ptr(blob), blob.size), entry.removeprefix("b2_"))

    def _new_lane(self, model: Optional[str], threaded: bool) -> _Lane:
        """Another library context on this device, configured like the front end's: its options are replayed first, because
        force_simt only applies to models loaded after it, then `model`'s weights are loaded (None: no model)."""
        ctx = _lib.Context(self.device.index)
        for name, value in self.ctx.options.items():
            ctx.set_option(name, value)
        if model is not None:
            self._set_weights(ctx, model)
        return _Lane(ctx, torch.cuda.Stream(self.device), ThreadPoolExecutor(max_workers=1) if threaded else None)

    def _role_lanes(self, model: str, n: int, threaded: bool = False) -> List[_Lane]:
        """The first `n` lanes that run `model`, made on first use (with a host thread each if the role is `threaded`).  Lane 0
        is the front end's own context on the caller's stream."""
        with self._lane_lock:
            lanes = self._lanes[model]
            while len(lanes) < n:
                lanes.append(self._new_lane(model, threaded) if lanes else
                             _Lane(self.ctx, pool=ThreadPoolExecutor(max_workers=1) if threaded else None))
            return lanes[:n]

    def _verify_lane(self) -> _Lane:
        with self._lane_lock:
            if self._vlane is None:
                # the matcher's persistent kernels (one CTA per SM) leave a few SMs to the concurrent RANSAC kernels: a CTA
                # that finds its SM occupied would wait for a whole CTA lifetime and double the kernel's duration
                self._set_option("reserve_sms", RESERVE_SMS_FOR_VERIFY)
                self._vlane = self._new_lane(None, threaded=True)
            return self._vlane

    def _set_option(self, name: str, value: int) -> None:
        """b2_set_option on the front end's context and on every lane made so far; lanes made later get it by the replay."""
        with self._lane_lock:
            for ctx in self._all_ctx() + ([self._vlane.ctx] if self._vlane is not None else []):
                ctx.set_option(name, value)

    @property
    def _vctx(self) -> Optional[_lib.Context]:
        """The verification lane's context, None until verification has been used."""
        return self._vlane.ctx if self._vlane is not None else None

    # measurement helpers over every context that runs SuperPoint / matcher kernels for this front end (bench.py)
    def _all_ctx(self):
        return [self.ctx] + [lane.ctx for lanes in self._lanes.values() for lane in lanes[1:]]

    def launch_count(self) -> int:
        return sum(c.launch_count() for c in self._all_ctx())

    def profile_start(self, kernel_prefix: str) -> None:
        for c in self._all_ctx():
            c.profile_start(kernel_prefix)

    def profile_stop(self):
        ms, n, w = 0.0, 0, 0.0
        for c in self._all_ctx():
            a, b, d = c.profile_stop()
            ms, n, w = ms + a, n + b, w + d
        return ms, n, w

    def _stream(self):
        return _lib.C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def ingest(self, image: torch.Tensor, max_resolution: int = 760) -> torch.Tensor:
        """Loader-side down-size on the device (gtsfm/loader/loader_base.py:160-200 -> gtsfm/utils/images.py:102-129,150-220):
        uint8 (H, W[, C]) device tensor -> cubic resize so that the short side is `max_resolution` (unchanged if already smaller)."""
        assert image.dtype == torch.uint8 and image.is_cuda and image.is_contiguous()
        h, w = int(image.shape[0]), int(image.shape[1])
        ch = 1 if image.dim() == 2 else int(image.shape[2])
        if min(h, w) <= max_resolution:
            return image
        if h <= w:
            nh, nw = max_resolution, int(np.round(w * (max_resolution / float(h))).astype(np.int32))
        else:
            nh, nw = int(np.round(h * (max_resolution / float(w))).astype(np.int32)), max_resolution
        out = torch.empty((nh, nw) if image.dim() == 2 else (nh, nw, ch), dtype=torch.uint8, device=self.device)
        rc = self.lib.b2_image_resize_dev(self.ctx.handle, _lib.ptr(image), h, w, ch, w * ch, _lib.ptr(out), nh, nw, self._stream())
        self.ctx.check(rc, "image_resize_dev")
        return out

    def ingest_jpeg(self, datas: Sequence[bytes], max_resolution: int = 760) -> List[torch.Tensor]:
        """JPEG file bytes -> device RGB frames (the pixels PIL would give, image_io.JpegEngine) -> `ingest`'s cubic down-size:
        a loader's files reach `detect` / `detect_many` without the pixels touching the host.  ValueError for a file the
        device decoder does not accept."""
        if getattr(self, "_jpeg", None) is None:
            from .image_io import JpegEngine

            self._jpeg = JpegEngine(self.device.index, ctx=self.ctx)
        return [self.ingest(f, max_resolution) for f in self._jpeg.decode_many(datas)]

    def detect(self, image: torch.Tensor, mask: Optional[np.ndarray] = None) -> DeviceFeatures:
        """image: uint8 device tensor (H, W) or (H, W, 3|4), contiguous.  One C call (detect -> device top-k -> describe): no
        torch kernels on the path, and the dense map never outlives the call (interleaving images on one handle is safe).
        `mask` (host (H, W) array, 1 = keep; gtsfm/common/keypoints.py:112-127) is applied BEFORE the top-k like the
        reference wrapper does (gtsfm/.../superpoint.py:87-91); masked images take the two-call path."""
        assert image.dtype == torch.uint8 and image.is_cuda and image.is_contiguous()
        h, w = int(image.shape[0]), int(image.shape[1])
        ch = 1 if image.dim() == 2 else int(image.shape[2])
        if mask is not None:
            return self._detect_masked(image, h, w, ch, np.asarray(mask))
        k = self.max_keypoints
        kp = torch.empty((k, 2), dtype=torch.float32, device=self.device)
        score = torch.empty(k, dtype=torch.float32, device=self.device)
        desc = torch.empty((k, 256), dtype=torch.float32, device=self.device)
        n = _lib.C.c_int(0)
        rc = self.lib.b2_superpoint_extract_dev(self.ctx.handle, _lib.ptr(image), h, w, ch, w * ch, KEYPOINT_THRESHOLD, NMS_RADIUS,
                                                REMOVE_BORDERS, k, _lib.ptr(kp), _lib.ptr(score), _lib.ptr(desc), _lib.C.byref(n),
                                                self._stream())
        self.ctx.check(rc, "superpoint_extract_dev")
        return DeviceFeatures(kp[: n.value], score[: n.value], desc[: n.value], (h, w))

    def detect_many(self, images) -> list:
        """`detect` for a list of images with every image enqueued before the first result is read: no host synchronisation
        between images (b2_superpoint_extract_async_dev), one at the end (b2_superpoint_finish_dev).  Images alternate between
        DETECT_LANES lanes (library contexts configured like the front end's) on as many streams, so one image's narrow kernels
        (80-CTA layers, the one-block top-k / scan) and launch gaps are filled by the other's.  Same outputs as
        [detect(im) for im in images]."""
        if len(images) == 0:
            return []
        kp_all, score_all, desc_all, counts, shapes = self.detect_pool(images)
        return [DeviceFeatures(kp_all[i, :n], score_all[i, :n], desc_all[i, :n], shapes[i]) for i, n in enumerate(counts)]

    def detect_pool(self, images, slots: Optional[int] = None):
        """detect_many's engine: -> (kp (slots, k, 2), score (slots, k), desc (slots, k, 256) device tensors, counts list, shapes);
        image i fills slot i (`slots` >= len(images): padding slots for the multi-GPU feature exchange)."""
        k = self.max_keypoints
        if self._counts is None or self._counts.numel() < len(images):  # page-locked once, reused (cudaHostAlloc is slow)
            self._counts = torch.zeros(max(64, len(images)), dtype=torch.int32).pin_memory()
        counts = self._counts
        outs = []
        lanes = self._role_lanes("superpoint", min(DETECT_LANES, max(1, len(images))))
        main = torch.cuda.current_stream(self.device)
        streams = [main] + [lane.stream for lane in lanes[1:]]
        # ONE allocation per output kind for the whole list (a fresh 5 MB descriptor block per image is a cudaMalloc each when the
        # caller keeps every image's features alive: 360 of them cost 0.7 s for 120 frames), sliced per image
        nimg = max(len(images), slots or 0)
        kp_all = torch.empty((nimg, k, 2), dtype=torch.float32, device=self.device)
        score_all = torch.empty((nimg, k), dtype=torch.float32, device=self.device)
        desc_all = torch.empty((nimg, k, 256), dtype=torch.float32, device=self.device)
        for stream in streams[1:]:
            # the images, and the previous owner of the output blocks (caching allocator), are done on the caller's stream
            stream.wait_stream(main)
            for t in (kp_all, score_all, desc_all):
                t.record_stream(stream)
        for i, image in enumerate(images):
            assert image.dtype == torch.uint8 and image.is_cuda and image.is_contiguous()
            ctx, stream = lanes[i % len(lanes)].ctx, streams[i % len(lanes)]
            h, w = int(image.shape[0]), int(image.shape[1])
            ch = 1 if image.dim() == 2 else int(image.shape[2])
            kp, score, desc = kp_all[i], score_all[i], desc_all[i]
            rc = self.lib.b2_superpoint_extract_async_dev(ctx.handle, _lib.ptr(image), h, w, ch, w * ch, KEYPOINT_THRESHOLD,
                                                          NMS_RADIUS, REMOVE_BORDERS, k, _lib.ptr(kp), _lib.ptr(score), _lib.ptr(desc),
                                                          _lib.C.c_void_p(counts.data_ptr() + 4 * i), _lib.C.c_void_p(stream.cuda_stream))
            ctx.check(rc, "superpoint_extract_async_dev")
            outs.append((h, w))
        for lane, stream in zip(lanes, streams):
            lane.ctx.check(self.lib.b2_superpoint_finish_dev(lane.ctx.handle, _lib.C.c_void_p(stream.cuda_stream)), "superpoint_finish_dev")
        return kp_all, score_all, desc_all, counts[: len(images)].tolist(), outs

    def _detect_masked(self, image: torch.Tensor, h: int, w: int, ch: int, mask: np.ndarray) -> DeviceFeatures:
        cap = SuperPointEngine.capacity(h, w)
        xy = torch.empty((cap, 2), dtype=torch.float32, device=self.device)
        sc = torch.empty(cap, dtype=torch.float32, device=self.device)
        n, tok = _lib.C.c_int(0), _lib.C.c_uint64(0)
        rc = self.lib.b2_superpoint_detect_dev(self.ctx.handle, _lib.ptr(image), h, w, ch, w * ch, KEYPOINT_THRESHOLD, NMS_RADIUS,
                                               REMOVE_BORDERS, _lib.ptr(xy), _lib.ptr(sc), cap, _lib.C.byref(n), _lib.C.byref(tok),
                                               self._stream())
        self.ctx.check(rc, "superpoint_detect_dev")
        nk = min(n.value, cap)
        hxy, hsc = xy[:nk].cpu().numpy(), sc[:nk].cpu().numpy()
        r = np.round(hxy).astype(int)
        keep = np.flatnonzero(mask[r[:, 1], r[:, 0]] == 1)
        if len(keep) > self.max_keypoints:  # the k largest responses, ties by lower index, row-major order kept
            keep = np.sort(keep[np.argsort(-hsc[keep], kind="stable")[: self.max_keypoints]])
        kp = torch.from_numpy(np.ascontiguousarray(hxy[keep])).to(self.device)
        score = torch.from_numpy(np.ascontiguousarray(hsc[keep])).to(self.device)
        desc = torch.empty((len(keep), 256), dtype=torch.float32, device=self.device)
        rc = self.lib.b2_superpoint_describe_dev(self.ctx.handle, tok.value, _lib.ptr(kp), len(keep), _lib.ptr(desc), self._stream())
        self.ctx.check(rc, "superpoint_describe_dev")
        return DeviceFeatures(kp, score, desc, (h, w))

    def match(self, a: DeviceFeatures, b: DeviceFeatures, depth_confidence=0.95, width_confidence=0.99, filter_threshold=0.1):
        cap = max(1, min(len(a), len(b)))
        out = torch.empty((cap, 2), dtype=torch.int64, device=self.device)
        k, stop = _lib.C.c_int(0), _lib.C.c_int(0)
        prm = _lib.LightGlueParams(depth_confidence, width_confidence, filter_threshold, self.prune_min, self.fp16_attention)
        rc = self.lib.b2_lightglue_match_dev(self.ctx.handle, _lib.ptr(a.kp), _lib.ptr(a.desc), len(a), _lib.ptr(b.kp), _lib.ptr(b.desc),
                                             len(b), _lib.C.byref(prm), _lib.ptr(out), None, _lib.C.byref(k), _lib.C.byref(stop),
                                             self._stream())
        self.ctx.check(rc, "lightglue_match_dev")
        return out[: k.value], stop.value

    def match_superglue_many(self, pairs: Sequence[Tuple[DeviceFeatures, DeviceFeatures]], on_pair=None, **kw) -> List[torch.Tensor]:
        """`match_superglue` over a list of pairs, dealt round-robin to SG_LANES lanes (library contexts configured like the front
        end's, with their own SuperGlue instance, stream and host thread each): SuperGlue runs pair by pair with many narrow
        kernels (2000-keypoint GNN layers, one-block filters), which concurrent pairs fill.  `on_pair(index, matches)` is called
        from the lane's thread as a pair completes, with `matches` complete on the device.  Results in input order."""
        if len(pairs) == 0:
            return []
        lanes = self._role_lanes("superglue", max(1, min(SG_LANES, len(pairs))), threaded=True)
        main = torch.cuda.current_stream(self.device)

        def work(j):
            lane, res = lanes[j], []
            with torch.cuda.stream(lane.stream if lane.stream is not None else main):
                for i in range(j, len(pairs), len(lanes)):
                    m = self.match_superglue(*pairs[i], ctx=lane.ctx, **kw)
                    if lane.stream is not None:
                        m.record_stream(main)
                    if on_pair:
                        # match_superglue's int64 conversion is still queued on this lane's stream: complete it before
                        # `on_pair` can hand `m` to work on another stream (the verification lane)
                        torch.cuda.current_stream(self.device).synchronize()
                        on_pair(i, m)
                    res.append(m)
            return res

        for lane in lanes[1:]:
            lane.stream.wait_stream(main)  # the features were produced on the caller's stream
        out: List[Optional[torch.Tensor]] = [None] * len(pairs)
        for j, f in enumerate([lane.pool.submit(work, j) for j, lane in enumerate(lanes)]):
            out[j::len(lanes)] = f.result()
        return out  # type: ignore[return-value]

    def match_superglue(self, a: DeviceFeatures, b: DeviceFeatures, sinkhorn_iters: int = 20, match_threshold: float = 0.2,
                        ctx: Optional[_lib.Context] = None) -> torch.Tensor:
        """SuperGlue on device-resident features -> (k, 2) int64 device tensor (rows (i, matches0[i]) ascending in i)."""
        cap = max(1, min(len(a), len(b)))
        out = torch.empty((cap, 2), dtype=torch.int32, device=self.device)  # the ABI writes uint32 rows
        k = _lib.C.c_int(0)
        ctx = ctx or self.ctx
        rc = self.lib.b2_superglue_match_dev(ctx.handle, _lib.ptr(a.kp), _lib.ptr(a.score), _lib.ptr(a.desc), len(a), a.shape[0], a.shape[1],
                                             _lib.ptr(b.kp), _lib.ptr(b.score), _lib.ptr(b.desc), len(b), b.shape[0], b.shape[1],
                                             int(sinkhorn_iters), float(match_threshold), _lib.ptr(out), None, _lib.C.byref(k), self._stream())
        ctx.check(rc, "superglue_match_dev")
        return out[: k.value].to(torch.int64)

    def match_many(self, pairs: Sequence[Tuple[DeviceFeatures, DeviceFeatures]], on_chunk=None, **kw) -> List[Tuple[torch.Tensor, int]]:
        """`match_batch` over any number of pairs in lock-step batches of 8, every image encoded once up front (one LightGlue
        instance: the matcher's persistent kernels already fill the GPU, so concurrent instances measured no gain).
        `on_chunk(first_pair_index, results)` is called as soon as a batch is complete - the hook bench.py uses to start
        verification early.  Results in input order."""
        self.encode([f for p in pairs for f in p])
        out = []
        for c0 in range(0, len(pairs), 8):
            r = self.match_batch(pairs[c0:c0 + 8], **kw)
            if on_chunk:
                on_chunk(c0, r)
            out += r
        return out

    def match_batch(self, pairs: Sequence[Tuple[DeviceFeatures, DeviceFeatures]], depth_confidence=0.95, width_confidence=0.99,
                    filter_threshold=0.1) -> List[Tuple[torch.Tensor, int]]:
        """LightGlue over a list of pairs through `b2_lightglue_match_batched_dev`: the library walks up to 8 pairs in
        lock-step (one launch per layer step for all their images), starting every image from its encoding (`encode`).
        -> [(matches (k, 2) int64 device tensor, stop layer)]."""
        n = len(pairs)
        if n == 0:
            return []
        key = self.encode([f for p in pairs for f in p])
        arr = (_lib.LightGluePair * n)()
        outs = []
        for i, (a, b) in enumerate(pairs):
            out = torch.empty((max(1, min(len(a), len(b))), 2), dtype=torch.int64, device=self.device)
            outs.append(out)
            arr[i].kp0, arr[i].desc0, arr[i].n0, arr[i].enc0 = a.kp.data_ptr(), a.desc.data_ptr(), len(a), a.enc[key].data_ptr()
            arr[i].kp1, arr[i].desc1, arr[i].n1, arr[i].enc1 = b.kp.data_ptr(), b.desc.data_ptr(), len(b), b.enc[key].data_ptr()
            arr[i].out_matches, arr[i].out_scores = out.data_ptr(), None
        prm = _lib.LightGlueParams(depth_confidence, width_confidence, filter_threshold, self.prune_min, self.fp16_attention)
        rc = self.lib.b2_lightglue_match_batched_dev(self.ctx.handle, arr, n, _lib.C.byref(prm), self._stream())
        self.ctx.check(rc, "lightglue_match_batched_dev")
        return [(outs[i][: arr[i].out_k], int(arr[i].out_stop_layer)) for i in range(n)]

    def _enc_key(self) -> tuple:
        # an encoding holds layer-0 activations: valid only under the weights and kernel path (force_simt) of the front end
        # that made it, and under the attention numerics it was made with
        return self._serial, self.fp16_attention

    def encode(self, feats: Sequence[DeviceFeatures]) -> tuple:
        """Give every image in `feats` that has none its LightGlue encoding under this front end (the state after layer 0's
        self block, which does not depend on the partner image): one b2_lightglue_encode_batched_dev call on the current
        stream for all of them, so that an image matched against many partners runs that block once.  -> the encoding key."""
        key = self._enc_key()
        todo = list({id(f): f for f in feats if key not in f.enc}.values())
        if not todo:
            return key
        bufs = [torch.empty(int(self.lib.b2_lightglue_encoded_bytes(len(f))), dtype=torch.uint8, device=self.device) for f in todo]
        imgs = (_lib.LightGlueImage * len(todo))()
        for i, (f, buf) in enumerate(zip(todo, bufs)):
            imgs[i].kp, imgs[i].desc, imgs[i].n, imgs[i].out = f.kp.data_ptr(), f.desc.data_ptr(), len(f), buf.data_ptr()
        prm = _lib.LightGlueParams(0.0, 0.0, 0.0, self.prune_min, self.fp16_attention)
        self.ctx.check(self.lib.b2_lightglue_encode_batched_dev(self.ctx.handle, imgs, len(todo), _lib.C.byref(prm), self._stream()),
                       "lightglue_encode_batched_dev")
        for f, buf in zip(todo, bufs):
            f.enc[key] = buf
        return key

    def verify_async(self, a: DeviceFeatures, b: DeviceFeatures, matches: torch.Tensor, cal1, cal2, threshold_px: float = 4.0,
                     seed: int = DEFAULT_SEED):
        """Same as verify() but returns a concurrent.futures.Future; `matches` must already be complete on the device
        (match() synchronises its stream before returning)."""
        lane = self._verify_lane()
        return lane.pool.submit(self.verify, a, b, matches, cal1, cal2, threshold_px, seed, lane.ctx, lane.stream)

    def verify(self, a: DeviceFeatures, b: DeviceFeatures, matches: torch.Tensor, cal1: Sequence[float], cal2: Sequence[float],
               threshold_px: float = 4.0, seed: int = DEFAULT_SEED, ctx: Optional[_lib.Context] = None,
               stream: Optional[torch.cuda.Stream] = None):
        """cal = (f, u0, v0).  -> (E (3,3) | None, R, t, num_inliers, mask device tensor)."""
        ctx = ctx or self.ctx
        sptr = _lib.C.c_void_p(stream.cuda_stream) if stream is not None else self._stream()
        k = int(matches.shape[0])
        matches = matches.contiguous()  # kept alive in this frame until the C call has returned
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            mask = torch.zeros(max(k, 1), dtype=torch.uint8, device=self.device)  # zero-filled on the stream the kernels use
        if k < 6:  # opencv_verifier_base.py:70-79
            return None, None, None, 0, mask[:k]
        E, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
        c1, c2 = np.asarray(cal1, np.float64), np.asarray(cal2, np.float64)
        n = _lib.C.c_int(0)
        prm = _lib.RansacParams(threshold_px / max(c1[0], c2[0]), RANSAC_SUCCESS_PROB, E_MAX_ITERS, seed)
        rc = self.lib.b2_ransac_essential_dev(ctx.handle, _lib.ptr(a.kp), _lib.ptr(b.kp), _lib.ptr(matches), k, _lib.ptr(c1),
                                              _lib.ptr(c2), _lib.C.byref(prm), _lib.ptr(E), _lib.ptr(mask), _lib.C.byref(n), _lib.ptr(R),
                                              _lib.ptr(t), sptr)
        ctx.check(rc, "ransac_essential_dev")
        if rc == 1:
            return None, None, None, 0, mask[:k]
        return E.reshape(3, 3), R.reshape(3, 3), t, n.value, mask[:k]

    def verify_many_async(self, items: Sequence[tuple], threshold_px: float = 4.0, seed: int = DEFAULT_SEED, method: str = "ransac"):
        """Same as verify_many() but returns ONE concurrent.futures.Future for the whole list, run on the verification lane
        (its own context, stream and thread, under the matcher's kernels); every `matches` must already be complete on the
        device."""
        _check_method(method)
        lane = self._verify_lane()
        return lane.pool.submit(self.verify_many, items, threshold_px, seed, lane.ctx, lane.stream, method)

    def verify_many(self, items: Sequence[tuple], threshold_px: float = 4.0, seed: int = DEFAULT_SEED,
                    ctx: Optional[_lib.Context] = None, stream: Optional[torch.cuda.Stream] = None, method: str = "ransac") -> list:
        """verify() for a list of (a, b, matches, cal1, cal2) in one b2_ransac_verify_batched_dev call: every stage is
        launched once for all pairs and the call synchronises once.  -> the list of verify()'s tuples, equal to them bit
        for bit.  method="lmeds": cv2's LMeDS (the reference's LMEDS verifier, 5-point E) in one
        b2_lmeds_verify_batched_dev call instead; `threshold_px` and `seed` are not used there (LMeDS has neither)."""
        _check_method(method)
        ctx = ctx or self.ctx
        sptr = _lib.C.c_void_p(stream.cuda_stream) if stream is not None else self._stream()
        ks = [int(m.shape[0]) for _, _, m, _, _ in items]
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            masks = torch.zeros(sum(ks) + 1, dtype=torch.uint8, device=self.device)  # zero-filled on the stream the kernels use
        out, live, problems, keep, off = [], [], [], [], 0
        for (a, b, m, cal1, cal2), k in zip(items, ks):
            mask = masks[off:off + k]
            off += k
            out.append((None, None, None, 0, mask))
            if k < 6:  # opencv_verifier_base.py:70-79
                continue
            m = m.contiguous()
            keep.append(m)  # alive until the C call has returned
            live.append(len(out) - 1)
            thr = threshold_px / max(float(cal1[0]), float(cal2[0])) if method == "ransac" else 0.0
            problems.append(ransac_problem(k, 0, thr, E_MAX_ITERS if method == "ransac" else LMEDS_MAX_ITERS, mask=mask, kp1=a.kp,
                                           kp2=b.kp, matches=m, cal1=cal1, cal2=cal2))
        if not problems:
            return out
        arr = (_lib.RansacProblem * len(problems))(*problems)
        res = (_lib.RansacResult * len(problems))()
        if method == "ransac":
            prm = _lib.RansacParams(0.0, RANSAC_SUCCESS_PROB, 0, seed)
            ctx.check(self.lib.b2_ransac_verify_batched_dev(ctx.handle, arr, len(problems), _lib.C.byref(prm), res, sptr),
                      "ransac_verify_batched_dev")
        else:
            ctx.check(self.lib.b2_lmeds_verify_batched_dev(ctx.handle, arr, len(problems), _lib.C.byref(lmeds_params()), res, sptr),
                      "lmeds_verify_batched_dev")
        for i, r in zip(live, res):
            if r.status == 0:
                out[i] = (np.array(r.model).reshape(3, 3), np.array(r.R).reshape(3, 3), np.array(r.t), r.num_inliers, out[i][4])
        return out


    def refine_many_async(self, items: Sequence[tuple], verified, options: "RefineOptions"):
        """refine_many() queued on the verification lane behind the verification whose Future is `verified` (the lane's one
        host thread runs them in order, on the lane's stream): -> ONE Future for the whole list."""
        lane = self._verify_lane()
        return lane.pool.submit(lambda: self.refine_many(items, verified.result(), options, lane.ctx, lane.stream))

    def refine_many(self, items: Sequence[tuple], verified: Sequence[tuple], options: "RefineOptions",
                    ctx: Optional[_lib.Context] = None, stream: Optional[torch.cuda.Stream] = None, trace: bool = False,
                    out_masks: Optional[Sequence[Optional[torch.Tensor]]] = None) -> list:
        """The reference's triangulation, two-view bundle adjustment and inlier support (two_view_estimator.py:350-481
        with bundle_adjust_2view) for a list of (a, b, matches, cal1, cal2) and verify_many()'s results for them, in one
        b2_twoview_ba_batched_dev call.  -> per item (R (3, 3) | None, unit t | None, kept rows as a DEVICE (n, 2) int64
        tensor | None, the b2_twoview_result | None); None, None, None, None for a pair whose verification failed.
        `trace`: also the LM cost traces, [n][max_iters + 2] (the test-only entry point).  `out_masks[i]`: a DEVICE (k,)
        uint8 tensor that receives the rows bundle adjustment kept, before inlier support (the post-BA rows)."""
        ctx = ctx or self.ctx
        sptr = _lib.C.c_void_p(stream.cuda_stream) if stream is not None else self._stream()
        out: list = [(None, None, None, None)] * len(items)
        live, problems, keep = [], [], []
        with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
            for i, ((a, b, m, cal1, cal2), (E, R, t, _, mask)) in enumerate(zip(items, verified)):
                if E is None:
                    continue
                m = m.contiguous()
                rows = torch.empty((max(int(m.shape[0]), 1), 2), dtype=torch.int64, device=self.device)
                keep.append((m, rows))
                live.append(i)
                p = _lib.TwoViewProblem()
                p.kp1, p.kp2, p.matches, p.mask, p.out_rows = (_lib.ptr(x) for x in (a.kp, b.kp, m, mask, rows))
                if out_masks is not None and out_masks[i] is not None:
                    p.out_mask = _lib.ptr(out_masks[i])
                p.k = int(m.shape[0])
                p.cal1[:], p.cal2[:] = [float(c) for c in cal1], [float(c) for c in cal2]
                p.R[:], p.t[:] = [float(v) for v in np.asarray(R).ravel()], [float(v) for v in np.asarray(t).ravel()]
                problems.append(p)
        if not problems:
            return (out, None) if trace else out
        n = len(problems)
        arr = (_lib.TwoViewProblem * n)(*problems)
        res = (_lib.TwoViewResult * n)()
        prm = options.params()
        if trace:
            tr = np.zeros((n, prm.max_iters + 2))
            ctx.check(self.lib.b2_debug_twoview_ba_trace_host(ctx.handle, arr, n, _lib.C.byref(prm), res, _lib.ptr(tr), sptr),
                      "debug_twoview_ba_trace_host")
        else:
            ctx.check(self.lib.b2_twoview_ba_batched_dev(ctx.handle, arr, n, _lib.C.byref(prm), res, sptr), "twoview_ba_batched_dev")
        for j, (i, r) in enumerate(zip(live, res)):
            if r.status == 0:
                out[i] = (np.array(r.R).reshape(3, 3), np.array(r.t), keep[j][1][:r.num_rows], r)
            else:
                out[i] = (None, None, None, r)
        return (out, tr) if trace else out

    def evaluate_many_async(self, units_fn, threshold_px: float = 4.0):
        """evaluate_many() queued on the verification lane behind the work already queued there: `units_fn()` is called on
        the lane's thread (after the verification / refinement Futures it reads are done) and returns the units.  -> ONE
        Future for the whole list."""
        lane = self._verify_lane()
        return lane.pool.submit(lambda: self.evaluate_many(units_fn(), threshold_px, lane.ctx, lane.stream))

    def evaluate_many(self, units: Sequence["EvalUnit"], threshold_px: float = 4.0, ctx: Optional[_lib.Context] = None,
                      stream: Optional[torch.cuda.Stream] = None) -> list:
        """The ground-truth metrics of the two-view reports (two_view_estimator.py:290-344) for a list of (pair, stage)
        units in one b2_twoview_eval_batched_dev call (one launch).  -> per unit (b2_twoview_eval_result, squared Sampson
        distances (n,) float64 HOST tensor, inlier mask (n,) uint8 HOST tensor), n the unit's rows; the tensors are empty
        without ground truth.  The kernel writes the per-row results straight into page-locked host memory, so they are
        on the host when the call's one synchronisation returns: no copy of their own."""
        ctx = ctx or self.ctx
        sptr = _lib.C.c_void_p(stream.cuda_stream) if stream is not None else self._stream()
        if not units:
            return []
        ks = [int(u.matches.shape[0]) for u in units]
        d2 = torch.empty(sum(ks) + 1, dtype=torch.float64, pin_memory=True)
        inl = torch.empty(sum(ks) + 1, dtype=torch.uint8, pin_memory=True)
        arr = (_lib.TwoViewEvalProblem * len(units))()
        keep, off = [], 0
        for p, u, k in zip(arr, units, ks):
            m = u.matches.contiguous()
            keep.append(m)  # alive until the C call has returned
            p.kp1, p.kp2, p.matches, p.k = _lib.ptr(u.kp1), _lib.ptr(u.kp2), _lib.ptr(m), k
            p.mask = _lib.ptr(u.mask) if u.mask is not None else None
            if u.pose is not None:
                p.has_pose = 1
                p.R[:], p.t[:] = [float(v) for v in np.asarray(u.pose[0]).ravel()], [float(v) for v in np.asarray(u.pose[1]).ravel()]
            if u.cam1 is not None and u.cam2 is not None:
                p.has_gt = 1
                for (R, t, f, u0, v0), pr, pt, pc in ((u.cam1, p.wRi1, p.wti1, p.cal1), (u.cam2, p.wRi2, p.wti2, p.cal2)):
                    pr[:], pt[:] = [float(v) for v in np.asarray(R).ravel()], [float(v) for v in np.asarray(t).ravel()]
                    pc[:] = [float(f), float(u0), float(v0)]
            p.out_d2, p.out_inlier = d2.data_ptr() + 8 * off, inl.data_ptr() + off
            off += k
        res = (_lib.TwoViewEvalResult * len(units))()
        prm = _lib.TwoViewEvalParams(float(threshold_px))
        ctx.check(self.lib.b2_twoview_eval_batched_dev(ctx.handle, arr, len(units), _lib.C.byref(prm), res, sptr),
                  "twoview_eval_batched_dev")
        out, off = [], 0
        for r, k in zip(res, ks):
            n = r.num_rows if not r.no_gt else 0
            out.append((r, d2[off:off + n], inl[off:off + n]))
            off += k
        return out


@dataclass
class EvalUnit:
    """One (pair, stage) of the two-view reports' evaluation: the stage's rows are the rows of `matches` where `mask` is
    set (None: every row).  `pose` = (i2Ri1, i2ti1) of the stage or None; cam = (R_wTi, t_wTi, f, u0, v0) or None."""
    kp1: torch.Tensor
    kp2: torch.Tensor
    matches: torch.Tensor
    mask: Optional[torch.Tensor]
    pose: Optional[Tuple[np.ndarray, np.ndarray]]
    cam1: Optional[tuple]
    cam2: Optional[tuple]


@dataclass
class RefineOptions:
    """The two-view refinement's settings (gtsfm/two_view_estimator.py:86-99, inlier_support_processor.py, and the
    front-end configs' triangulation options)."""
    ba_reproj_error_threshold: float = 0.5
    min_num_inliers_est_model: int = 15
    min_inlier_ratio_est_model: float = 0.1
    triangulation_reproj_error_threshold: float = float("inf")
    min_triangulation_angle: float = 0.0
    max_iters: int = 100

    def params(self) -> "_lib.TwoViewParams":
        return _lib.TwoViewParams(int(self.max_iters), int(self.min_num_inliers_est_model), float(self.min_inlier_ratio_est_model),
                                  float(self.ba_reproj_error_threshold), float(self.triangulation_reproj_error_threshold),
                                  float(self.min_triangulation_angle))


def _check_method(method: str) -> None:
    if method not in ("ransac", "lmeds"):
        raise ValueError(f"verification method must be 'ransac' or 'lmeds', not {method!r}")


from .distributed import shard_pairs  # noqa: E402,F401  (re-export: `p mod world` partitioner)
