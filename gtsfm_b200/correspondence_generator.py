"""Batched, device-resident correspondence generator: the L2 seam of SURVEY.md §8b.

Implements `CorrespondenceGeneratorBase.generate_correspondences(client, images, visibility_graph)`
(gtsfm/frontend/correspondence_generator/correspondence_generator_base.py:19-36) without creating one Dask task per
image and per pair (det_desc_correspondence_generator.py:65-85): each image is detected once on the GPU, its features stay
in HBM, every pair of this process's shard is matched there, and only `(K, 2)` index arrays and keypoints come back.
Under `torch.distributed` (one process per GPU) the pair list is sharded `p mod world` and merged at the end.

One class serves every device detector (SuperPoint, SIFT, ORB, D2-Net) and matcher (LightGlue, SuperGlue, the two-way
matcher): what differs per detector is the `_DETECTORS` table, and what the generator returns equals what the matching
plugins of detector_descriptor.py and matcher.py return for the same images."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import distributed as D
from . import detector_descriptor as DD
from .gtsfm_api import HAVE_GTSFM, Keypoints
from .pipeline import DeviceFeatures, DeviceFrontEnd

if HAVE_GTSFM:  # pragma: no cover
    from gtsfm.frontend.correspondence_generator.correspondence_generator_base import CorrespondenceGeneratorBase as _Base
else:
    _Base = object


@dataclass(frozen=True)
class _Detector:
    engine: Optional[str]  # detector_descriptor engine whose extract_many detects a batch (None: DeviceFrontEnd.detect_many)
    desc_dtype: torch.dtype
    desc_dim: int
    scales: bool  # the plugin's Keypoints carry scales (the keypoint size) and float64 fields
    device_masks: bool  # extract_many applies image.mask on the device (D2-Net ignores masks, as its plugin does)


_DETECTORS = {"superpoint": _Detector(None, torch.float32, DD.DESC_DIM, False, False),
              "sift": _Detector("SiftEngine", torch.uint8, DD.SIFT_DESC_DIM, True, True),
              "orb": _Detector("OrbEngine", torch.uint8, DD.ORB_DESC_DIM, True, True),
              "d2net": _Detector("D2NetEngine", torch.float32, DD.D2NET_DESC_DIM, False, False)}
_MATCHERS = ("lightglue", "superglue", "twoway")
TWOWAY_CHUNK = 16  # pairs per b2_mnn_match_batched_dev call: each chunk's verification starts under the next chunk's matching
SUPERGLUE_CHUNK = 8  # SuperGlue pairs verified per call, in completion order


class B200CorrespondenceGenerator(_Base):
    """`detector`: "superpoint" | "sift" | "orb" | "d2net"; `matcher`: "lightglue" | "superglue" (both take SuperPoint's
    features) | "twoway" (any detector, with `ratio_test_threshold`).  Weights: `superpoint_weights`, `lightglue_weights`,
    `superglue_weights` and `d2net_weights` (default: the D2-Net plugin's default path) for the models chosen."""

    def __init__(self, superpoint_weights=None, lightglue_weights=None, max_keypoints: int = 5000, device: int = 0, cpu_semantics: bool = True,
                 detector: str = "superpoint", matcher: str = "lightglue", superglue_weights=None, d2net_weights=None,
                 ratio_test_threshold: Optional[float] = None):
        if detector not in _DETECTORS:
            raise ValueError(f"detector must be one of {sorted(_DETECTORS)}, not {detector!r}")
        if matcher not in _MATCHERS:
            raise ValueError(f"matcher must be one of {list(_MATCHERS)}, not {matcher!r}")
        if matcher != "twoway" and detector != "superpoint":
            raise ValueError(f"the {matcher} matcher takes SuperPoint features; use matcher='twoway' with {detector}")
        self._sp, self._lg, self._sg, self._d2 = superpoint_weights, lightglue_weights, superglue_weights, d2net_weights
        self._max_keypoints, self._device, self._cpu_semantics = max_keypoints, device, cpu_semantics
        self._detector, self._matcher, self._ratio = detector, matcher, ratio_test_threshold
        self._fe: Optional[DeviceFrontEnd] = None
        self._det_engine = None  # the detector's batched engine (SIFT / ORB / D2-Net), on the front end's context
        self._mnn = None  # the two-way matcher's engine, on the front end's context
        self.last_device_features: Dict[int, DeviceFeatures] = {}  # device-resident features of the last call (for the two-view seam)
        self.last_detections = 0  # images this rank detected in the last call
        self.last_two_view: Dict[Tuple[int, int], object] = {}  # {pair: TwoViewResult} of the last call with verify_with

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_fe"] = st["_det_engine"] = st["_mnn"] = None
        st["last_device_features"] = {}
        st["last_two_view"] = {}
        return st

    def _front_end(self) -> DeviceFrontEnd:
        if self._fe is None:
            sp = self._sp if self._detector == "superpoint" else None
            lg = self._lg if self._matcher == "lightglue" else None
            sg = self._sg if self._matcher == "superglue" else None
            self._fe = DeviceFrontEnd(sp, lg, device=self._device, max_keypoints=self._max_keypoints, cpu_semantics=self._cpu_semantics,
                                      superglue_sd=sg)
        return self._fe

    def _engine(self, fe: DeviceFrontEnd):
        if self._det_engine is None:
            cls = getattr(DD, _DETECTORS[self._detector].engine)
            if cls is DD.D2NetEngine:
                self._det_engine = cls(DD.default_d2net_model_path() if self._d2 is None else self._d2, ctx=fe.ctx)
            else:
                self._det_engine = cls(ctx=fe.ctx)
        return self._det_engine

    def _detect(self, fe: DeviceFrontEnd, items) -> Dict[int, DeviceFeatures]:
        """items: [(image index, uint8 device image, host mask or None)] -> {index: DeviceFeatures}."""
        det, k, feats = _DETECTORS[self._detector], fe.max_keypoints, {}
        if det.engine is None:
            plain = []
            for idx, dev, mask in items:
                if mask is not None:
                    feats[idx] = fe.detect(dev, mask=mask)  # masks are applied on the host before the top-k: two-call path
                else:
                    plain.append((idx, dev))
            for c0 in range(0, len(plain), 32):  # unmasked images: enqueued 32 at a time, no synchronisation between images
                chunk = plain[c0:c0 + 32]
                for (idx, _), f in zip(chunk, fe.detect_many([d for _, d in chunk])):
                    feats[idx] = f
            return feats
        eng, groups = self._engine(fe), {}
        for it in items:  # extract_many takes images of one shape (and splits them into calls of at most images_per_call)
            groups.setdefault(tuple(it[1].shape), []).append(it)
        for group in groups.values():
            devs = [dev for _, dev, _ in group]
            if det.device_masks:
                # the batched call reads an H x W mask through its pointer alone: check the shape here, as the plugin's host
                # call does (SiftEngine.detect_and_describe)
                if any(m is not None and np.shape(m)[:2] != tuple(dev.shape[:2]) for _, dev, m in group):
                    raise ValueError("mask must have the image's height and width")
                masks = [None if m is None else torch.from_numpy(np.ascontiguousarray(m)).to(fe.device) for _, _, m in group]
                out = eng.extract_many(devs, masks=masks, max_keypoints=k)
                for (idx, dev, _), (rec, desc, _) in zip(group, out):  # records [x, y, size, angle, response, octave bits]
                    feats[idx] = DeviceFeatures(rec[:, :2].contiguous(), rec[:, 4].contiguous(), desc, tuple(dev.shape[:2]),
                                                scale=rec[:, 2].contiguous())
            else:
                for (idx, dev, _), (xy, sc, desc, _) in zip(group, eng.extract_many(devs, max_keypoints=k)):
                    feats[idx] = DeviceFeatures(xy, sc, desc, tuple(dev.shape[:2]))
        return feats

    def _detect_slots(self, fe: DeviceFrontEnd, items, n_loc: int):
        """The feature exchange's padded layout: image j of `items` fills slot j of (n_loc, k, ...) tensors.  -> ([kp (n_loc, k,
        2), score (n_loc, k), desc (n_loc, k, D)] plus sizes (n_loc, k) for the detectors with scales, counts, (h, w) shapes)."""
        det, k = _DETECTORS[self._detector], fe.max_keypoints
        if det.engine is None:  # SuperPoint writes its detections straight into the slots
            if items:
                kp, sc, de, counts, shapes = fe.detect_pool([dev for _, dev, _ in items], slots=n_loc)
                return [kp, sc, de], counts, shapes
            return [torch.empty((n_loc, k, 2), dtype=torch.float32, device=fe.device),
                    torch.empty((n_loc, k), dtype=torch.float32, device=fe.device),
                    torch.empty((n_loc, k, det.desc_dim), dtype=det.desc_dtype, device=fe.device)], [], []
        slots = [torch.empty((n_loc, k, 2), dtype=torch.float32, device=fe.device),
                 torch.empty((n_loc, k), dtype=torch.float32, device=fe.device),
                 torch.empty((n_loc, k, det.desc_dim), dtype=det.desc_dtype, device=fe.device)]
        if det.scales:
            slots.append(torch.empty((n_loc, k), dtype=torch.float32, device=fe.device))
        counts, shapes = [], []
        got = self._detect(fe, items)
        for j, (idx, _, _) in enumerate(items):  # the engines write per-image outputs: each is copied into its slot, then freed
            f = got.pop(idx)
            for t, v in zip(slots, (f.kp, f.score, f.desc, f.scale)):
                t[j, :len(f)] = v
            counts.append(len(f))
            shapes.append(f.shape)
        return slots, counts, shapes

    def _match(self, fe: DeviceFrontEnd, pairs: Sequence[Tuple[DeviceFeatures, DeviceFeatures]], on_chunk) -> List[torch.Tensor]:
        """-> one (k, 2) int64 device tensor per pair; `on_chunk(pair indices, their matches)` runs as each chunk is complete."""
        if self._matcher == "lightglue":  # lock-step batches of 8 pairs (b2_lightglue_match_batched_dev), in order
            res = fe.match_many(pairs, on_chunk=lambda c0, r: on_chunk(range(c0, c0 + len(r)), [m for m, _ in r]))
            return [m for m, _ in res]
        if self._matcher == "superglue":  # pairs complete out of order on SG_LANES lanes: chunks of SUPERGLUE_CHUNK as they finish
            import threading

            lock, done = threading.Lock(), []

            def on_pair(i, m):
                with lock:
                    done.append((i, m))
                    if len(done) < SUPERGLUE_CHUNK:
                        return
                    chunk = done[:]
                    done.clear()
                on_chunk([i for i, _ in chunk], [m for _, m in chunk])

            out = fe.match_superglue_many(pairs, on_pair=on_pair)
            if done:
                on_chunk([i for i, _ in done], [m for _, m in done])
            return out
        if self._mnn is None:
            from .matcher import TwoWayEngine

            self._mnn = TwoWayEngine(ctx=fe.ctx)
        out: List[torch.Tensor] = []
        for c0 in range(0, len(pairs), TWOWAY_CHUNK):
            chunk = pairs[c0:c0 + TWOWAY_CHUNK]
            ms = [torch.empty((0, 2), dtype=torch.int64, device=fe.device)] * len(chunk)
            live = [j for j, (a, b) in enumerate(chunk) if len(a) and len(b)]  # an image without keypoints matches nothing
            for j, m in zip(live, self._mnn.match_batched_dev([(chunk[j][0].desc, chunk[j][1].desc) for j in live], self._ratio)):
                ms[j] = m
            on_chunk(range(c0, c0 + len(chunk)), ms)
            out += ms
        return out

    def _host_matches(self, m: torch.Tensor) -> np.ndarray:
        """Device rows -> the array the matcher's plugin returns: int64 (LightGlue), uint32 (SuperGlue), uint32 or, without a
        match, np.array([]) (the two-way matcher, twoway_matcher.py:72-73)."""
        h = m.cpu().numpy()
        if self._matcher == "lightglue":
            return h
        if self._matcher == "twoway" and len(h) == 0:
            return np.array([])
        return h.astype(np.uint32)

    def _keypoints(self, f: DeviceFeatures) -> Keypoints:
        """The Keypoints the detector's plugin returns: float64 (x, y), sizes and responses for SIFT / ORB (and a bare
        Keypoints for an image without keypoints), float32 (x, y) and responses for SuperPoint / D2-Net."""
        if not _DETECTORS[self._detector].scales:
            return Keypoints(f.kp.cpu().numpy(), scales=None, responses=f.score.cpu().numpy())
        if len(f) == 0:
            return Keypoints(np.zeros((0, 2)))
        return Keypoints(f.kp.cpu().numpy().astype(np.float64), scales=f.scale.cpu().numpy().astype(np.float64),
                         responses=f.score.cpu().numpy().astype(np.float64))

    def generate_correspondences(self, client, images: Sequence, visibility_graph: Sequence[Tuple[int, int]], verify_with=None):
        """-> (List[Keypoints] per image, Dict[(i1, i2), (K, 2) match rows in the matcher plugin's dtype]).

        `verify_with = (intrinsics {image: (f, u0, v0)}, threshold_px)` additionally runs the two-view verification of this
        rank's pairs (gtsfm/two_view_estimator.py:350-481) UNDER the matching - a chunk's RANSAC is queued on the verification
        stream the moment its matches exist - and leaves {pair: TwoViewResult} in `self.last_two_view`.  An optional third
        element, a dict of B200TwoViewBatch's refinement arguments (`bundle_adjust_2view=True`, thresholds), also runs the
        triangulation, two-view bundle adjustment and inlier support right behind each chunk's verification."""
        import time

        t_start = time.perf_counter()
        fe = self._front_end()
        det = _DETECTORS[self._detector]
        rank = torch.distributed.get_rank() if torch.distributed.is_initialized() else 0
        world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1
        mine = D.shard_pairs(list(visibility_graph), rank, world)
        feats: Dict[int, DeviceFeatures] = {}

        def host_image(idx):
            img = images[idx].result() if hasattr(images[idx], "result") else images[idx]  # Dask Future or Image
            return img, (img.value_array if hasattr(img, "value_array") else np.asarray(img))

        def item(idx, img, arr):
            mask = getattr(img, "mask", None) if det.engine is None or det.device_masks else None
            return idx, torch.from_numpy(np.ascontiguousarray(arr)).to(fe.device), mask

        # only SuperPoint applies masks on the host (two calls per image); SIFT and ORB apply them inside the batched call
        host_masks = det.engine is None
        masked = host_masks and any(getattr(im, "mask", None) is not None for im in images if not hasattr(im, "result"))
        own = [i for i in range(len(images)) if D.image_owner(i, world) == rank]
        own_host = []
        if world > 1:
            own_host = [host_image(i) for i in own]
            if host_masks:
                # whether any image carries a mask must be decided by ALL ranks together (the branches below contain
                # different collectives): each rank looks at the images it owns (Dask futures resolve here)
                flag = torch.tensor([1 if masked or any(getattr(img, "mask", None) is not None for img, _ in own_host) else 0],
                                    dtype=torch.int32, device=fe.device)
                torch.distributed.all_reduce(flag, op=torch.distributed.ReduceOp.MAX)
                masked = bool(int(flag.item()))
        if world > 1 and not masked:
            # ONE job over several GPUs: every image is detected on exactly one rank (position mod world) and the features are
            # exchanged with one all-gather over NVLink (5 MB per SuperPoint image) - re-detecting on every rank whose pairs
            # touch an image made detection the part of the job that did not scale
            n_loc = (len(images) + world - 1) // world
            slots, counts, shapes = self._detect_slots(fe, [item(i, img, arr) for i, (img, arr) in zip(own, own_host)], n_loc)
            meta = torch.zeros((n_loc, 3), dtype=torch.int32, device=fe.device)  # (count, height, width) per slot
            if counts:
                meta[: len(counts)] = torch.tensor([[c, h, w] for c, (h, w) in zip(counts, shapes)], dtype=torch.int32)
            *gathered, meta_a = D.all_gather_features(*slots, meta)
            meta_h = meta_a.cpu().tolist()
            for i in range(len(images)):
                slot = D.image_owner(i, world) * n_loc + i // world
                c, h, w = meta_h[slot]
                kp_a, sc_a, de_a = (t[slot, :c] for t in gathered[:3])
                feats[i] = DeviceFeatures(kp_a, sc_a, de_a, (h, w), scale=gathered[3][slot, :c] if det.scales else None)
            self.last_detections = len(own)
        else:
            # images of this rank's pairs, plus (so that every image gets keypoints) images no pair references: idx mod world
            todo = set(range(len(images))) if world == 1 else set(D.images_needed(mine))
            if world > 1:
                paired = {i for p in visibility_graph for i in p}
                todo |= {i for i in range(len(images)) if i not in paired and i % world == rank}
            feats = self._detect(fe, [item(idx, *host_image(idx)) for idx in sorted(todo)])
            self.last_detections = len(todo)
        t_detect = time.perf_counter()
        local: Dict[Tuple[int, int], np.ndarray] = {}
        pending = []
        refine = None
        if verify_with is not None:
            from .two_view import B200TwoViewBatch, submit_chunk
            from .verifier import DEFAULT_SEED

            if len(verify_with) > 2:
                refine = B200TwoViewBatch(fe, **verify_with[2]).refine

        def on_chunk(idx, ms):  # a chunk of this rank's pairs whose matches are complete on the device
            if verify_with is None:
                return
            intr, thr = verify_with[:2]  # the chunk is verified by one batched call (pairs under 6 matches fail inside it)
            prs = [mine[j] for j in idx]
            items = [(feats[i1], feats[i2], m, intr[i1], intr[i2]) for (i1, i2), m in zip(prs, ms)]
            pending.append(submit_chunk(fe, prs, items, thr, DEFAULT_SEED, "ransac", refine))

        matched = self._match(fe, [(feats[i1], feats[i2]) for i1, i2 in mine], on_chunk)
        for f in feats.values():  # the matcher's per-image encodings (11.5 MB at 5000 keypoints) are not needed past matching
            f.enc.clear()
        t_match = time.perf_counter()
        for pair, m in zip(mine, matched):
            local[pair] = self._host_matches(m)
        if verify_with is not None:
            self.last_two_view = {}
            for chunk in pending:
                B200TwoViewBatch._collect_chunk(chunk, self.last_two_view)
        t_verify = time.perf_counter()
        self.last_device_features = feats
        matches = D.gather_pair_results(local)
        keypoints: List[Optional[Keypoints]] = [None] * len(images)
        for idx, f in feats.items():
            keypoints[idx] = self._keypoints(f)
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
