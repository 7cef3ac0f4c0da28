"""Multi-GPU plumbing for the pair-sharded front-end (SURVEY.md §8e): one process per GPU, `torch.distributed` for one weight
broadcast at start-up, one gather of the (small) per-pair results at the end and - when ONE job is split over the GPUs (strong
scaling) - one all-gather of the detected features, the path's only real exchange: every image is detected on exactly one
rank and its (keypoints, scores, descriptors) travel over NVLink (5 MB per image) instead of being re-detected by every rank
whose pairs touch it.  No collective on the per-pair path.  Backend-agnostic (NCCL on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

Pair = Tuple[int, int]


def shard_pairs(pairs: Sequence[Pair], rank: int, world: int) -> List[Pair]:
    """Pair p (in visibility-graph order) -> rank p mod world."""
    return [p for i, p in enumerate(pairs) if i % world == rank]


def images_needed(pairs: Sequence[Pair]) -> List[int]:
    """Images a rank must detect for its shard (re-detection is cheaper than exchanging features, SURVEY.md §8e(b))."""
    return sorted({i for p in pairs for i in p})


def image_owner(position: int, world: int) -> int:
    """The rank that detects the image at `position` of the sorted list of images to detect."""
    return position % world


def all_gather_features(*tensors: torch.Tensor):
    """Each rank passes the features of the images it detected, padded to the same shapes on every rank, one slot per image:
    e.g. kp (n, k, 2), score (n, k), desc (n, k, D) in the detector's dtype, counts (n,) int32 (0 for padding slots).  Returns
    the rank-major concatenations (world * n, ...) in the same order: slot r * n + j = rank r's j-th image."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return tensors
    world = dist.get_world_size()
    out = []
    for t in tensors:
        t = t.contiguous()
        full = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(full, t)
        out.append(full)
    return tuple(out)


def broadcast_state_dict(sd: Dict[str, np.ndarray], order: Sequence[str], src: int = 0, device: str = "cpu") -> Dict[str, np.ndarray]:
    """Rank `src` owns the weights; everyone leaves with identical copies.  One broadcast of one packed fp32 blob."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return sd
    shapes = [tuple(np.asarray(sd[k]).shape) for k in order]
    total = int(sum(int(np.prod(s)) if s else 1 for s in shapes))
    if dist.get_rank() == src:
        blob = torch.from_numpy(np.concatenate([np.asarray(sd[k], np.float32).ravel() for k in order])).to(device)
    else:
        blob = torch.empty(total, dtype=torch.float32, device=device)
    dist.broadcast(blob, src)
    flat = blob.cpu().numpy()
    out, off = dict(sd), 0
    for k, s in zip(order, shapes):
        n = int(np.prod(s)) if s else 1
        out[k] = flat[off:off + n].reshape(s).copy()
        off += n
    return out


def gather_pair_results(local: Dict[Pair, np.ndarray]) -> Dict[Pair, np.ndarray]:
    """Union of every rank's {pair: match array}; each pair is produced by exactly one rank."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return dict(local)
    parts: List[Dict[Pair, np.ndarray]] = [None] * dist.get_world_size()  # type: ignore[list-item]
    dist.all_gather_object(parts, local)
    merged: Dict[Pair, np.ndarray] = {}
    for part in parts:
        for k, v in part.items():
            assert k not in merged, f"pair {k} produced by two ranks"
            merged[k] = v
    return merged
