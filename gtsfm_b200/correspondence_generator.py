"""Batched, device-resident correspondence generator: the L2 seam of SURVEY.md §8b.

Implements `CorrespondenceGeneratorBase.generate_correspondences(client, images, visibility_graph)`
(gtsfm/frontend/correspondence_generator/correspondence_generator_base.py:19-36) without creating one Dask task per
image and per pair (det_desc_correspondence_generator.py:65-85): each image is detected once on the GPU, its features stay
in HBM, every pair of this process's shard is matched there, and only `(K, 2)` index arrays and keypoints come back.
Under `torch.distributed` (one process per GPU) the pair list is sharded `p mod world` and merged at the end."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import distributed as D
from .gtsfm_api import HAVE_GTSFM, Keypoints
from .pipeline import DeviceFeatures, DeviceFrontEnd

if HAVE_GTSFM:  # pragma: no cover
    from gtsfm.frontend.correspondence_generator.correspondence_generator_base import CorrespondenceGeneratorBase as _Base
else:
    _Base = object


class B200CorrespondenceGenerator(_Base):
    def __init__(self, superpoint_weights, lightglue_weights, max_keypoints: int = 5000, device: int = 0, cpu_semantics: bool = True):
        self._sp, self._lg = superpoint_weights, lightglue_weights
        self._max_keypoints, self._device, self._cpu_semantics = max_keypoints, device, cpu_semantics
        self._fe: Optional[DeviceFrontEnd] = None
        self.last_device_features: Dict[int, DeviceFeatures] = {}  # device-resident features of the last call (for the two-view seam)
        self.last_detections = 0  # images this rank detected in the last call
        self.last_two_view: Dict[Tuple[int, int], object] = {}  # {pair: TwoViewResult} of the last call with verify_with

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_fe"] = None
        st["last_device_features"] = {}
        st["last_two_view"] = {}
        return st

    def _front_end(self) -> DeviceFrontEnd:
        if self._fe is None:
            self._fe = DeviceFrontEnd(self._sp, self._lg, device=self._device, max_keypoints=self._max_keypoints,
                                      cpu_semantics=self._cpu_semantics)
        return self._fe

    def generate_correspondences(self, client, images: Sequence, visibility_graph: Sequence[Tuple[int, int]], verify_with=None):
        """-> (List[Keypoints] per image, Dict[(i1, i2), (K, 2) int64 match rows]).

        `verify_with = (intrinsics {image: (f, u0, v0)}, threshold_px)` additionally runs the two-view verification of this
        rank's pairs (gtsfm/two_view_estimator.py:350-481) UNDER the matching - a batch's RANSAC is queued on the verification
        stream the moment its matches exist - and leaves {pair: TwoViewResult} in `self.last_two_view`."""
        import time

        t_start = time.perf_counter()
        fe = self._front_end()
        rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
        world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        mine = D.shard_pairs(list(visibility_graph), rank, world)
        feats: Dict[int, DeviceFeatures] = {}

        def host_image(idx):
            img = images[idx].result() if hasattr(images[idx], "result") else images[idx]  # Dask Future or Image
            return img, (img.value_array if hasattr(img, "value_array") else np.asarray(img))

        masked = any(getattr(im, "mask", None) is not None for im in images if not hasattr(im, "result"))
        own = [i for i in range(len(images)) if D.image_owner(i, world) == rank]
        own_host = []
        if world > 1:
            # masks take the host two-call path, and whether any image carries one must be decided by ALL ranks together (the
            # branches below contain different collectives): each rank looks at the images it owns (Dask futures resolve here)
            own_host = [host_image(i) for i in own]
            flag = torch.tensor([1 if masked or any(getattr(img, "mask", None) is not None for img, _ in own_host) else 0],
                                dtype=torch.int32, device=fe.device)
            torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MAX)
            masked = bool(int(flag.item()))
        if world > 1 and not masked:
            # ONE job over several GPUs: every image is detected on exactly one rank (position mod world) and the features are
            # exchanged with one all-gather over NVLink (5 MB per image) - re-detecting on every rank whose pairs touch an image
            # made detection the part of the job that did not scale
            k = fe.max_keypoints
            n_loc = (len(images) + world - 1) // world
            devs = [torch.from_numpy(np.ascontiguousarray(arr)).to(fe.device) for _, arr in own_host]
            if devs:
                kp_l, sc_l, de_l, cnt, shapes = fe.detect_pool(devs, slots=n_loc)
            else:
                kp_l = torch.empty((n_loc, k, 2), dtype=torch.float32, device=fe.device)
                sc_l = torch.empty((n_loc, k), dtype=torch.float32, device=fe.device)
                de_l = torch.empty((n_loc, k, 256), dtype=torch.float32, device=fe.device)
                cnt, shapes = [], []
            meta = torch.zeros((n_loc, 3), dtype=torch.int32, device=fe.device)  # (count, height, width) per slot
            if cnt:
                meta[: len(cnt)] = torch.tensor([[c, h, w] for c, (h, w) in zip(cnt, shapes)], dtype=torch.int32)
            kp_a, sc_a, de_a, meta_a = D.all_gather_features(kp_l, sc_l, de_l, meta)
            meta_h = meta_a.cpu().tolist()
            for i in range(len(images)):
                slot = D.image_owner(i, world) * n_loc + i // world
                c, h, w = meta_h[slot]
                feats[i] = DeviceFeatures(kp_a[slot, :c], sc_a[slot, :c], de_a[slot, :c], (h, w))
            self.last_detections = len(own)
        else:
            # images of this rank's pairs, plus (so that every image gets keypoints) images no pair references: idx mod world
            todo = set(range(len(images))) if world == 1 else set(D.images_needed(mine))
            if world > 1:
                paired = {i for p in visibility_graph for i in p}
                todo |= {i for i in range(len(images)) if i not in paired and i % world == rank}
            plain: List[Tuple[int, torch.Tensor]] = []
            for idx in sorted(todo):
                img, arr = host_image(idx)
                dev = torch.from_numpy(np.ascontiguousarray(arr)).to(fe.device)
                if getattr(img, "mask", None) is not None:
                    feats[idx] = fe.detect(dev, mask=img.mask)  # masks are applied on the host before the top-k: two-call path
                else:
                    plain.append((idx, dev))
            for c0 in range(0, len(plain), 32):  # unmasked images: enqueued 32 at a time, no synchronisation between images
                chunk = plain[c0:c0 + 32]
                for (idx, _), f in zip(chunk, fe.detect_many([d for _, d in chunk])):
                    feats[idx] = f
            self.last_detections = len(todo)
        t_detect = time.perf_counter()
        local: Dict[Tuple[int, int], np.ndarray] = {}
        pending = []

        def on_chunk(c0, res):  # lock-step batches of 8 pairs (b2_lightglue_match_batched_dev), in completion order
            if verify_with is None:
                return
            intr, thr = verify_with  # the chunk is verified by one batched call (pairs under 6 matches fail inside it)
            prs = mine[c0:c0 + len(res)]
            items = [(feats[i1], feats[i2], m, intr[i1], intr[i2]) for (i1, i2), (m, _) in zip(prs, res)]
            pending.append((prs, [m for m, _ in res], fe.verify_many_async(items, thr)))

        matched = fe.match_many([(feats[i1], feats[i2]) for i1, i2 in mine], on_chunk=on_chunk)
        for f in feats.values():  # the matcher's per-image encodings (11.5 MB at 5000 keypoints) are not needed past matching
            f.enc.clear()
        t_match = time.perf_counter()
        for (i1, i2), (m, _) in zip(mine, matched):
            local[(i1, i2)] = m.cpu().numpy()
        if verify_with is not None:
            from .two_view import B200TwoViewBatch

            self.last_two_view = {}
            for chunk in pending:
                B200TwoViewBatch._collect_chunk(chunk, self.last_two_view)
        t_verify = time.perf_counter()
        self.last_device_features = feats
        matches = D.gather_pair_results(local)
        keypoints: List[Optional[Keypoints]] = [None] * len(images)
        for idx, f in feats.items():
            keypoints[idx] = Keypoints(f.kp.cpu().numpy(), scales=None, responses=f.score.cpu().numpy())
        if world > 1 and masked:  # every rank returns the keypoints of all images, like the reference's gather (:83-85);
            # after the feature exchange every rank already holds them all (`masked` is identical on all ranks: same image list)
            parts: List[Dict[int, Keypoints]] = [None] * world  # type: ignore[list-item]
            torch.distributed.all_gather_object(parts, {i: k for i, k in enumerate(keypoints) if k is not None})
            for part in parts:
                for i, k in part.items():
                    if keypoints[i] is None:  # (an empty Keypoints is falsy: test identity, not truth)
                        keypoints[i] = k
        t_end = time.perf_counter()
        self.last_timing = {"detect_s": t_detect - t_start, "match_s": t_match - t_detect, "collect_verify_s": t_verify - t_match,
                            "gather_s": t_end - t_verify}  # where a call's wall time went (bench.py --scaling strong reports it)
        return keypoints, matches
